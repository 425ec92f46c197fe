#!/usr/bin/env python
"""Time one ``Agent.learn`` at batch 64 as the trainer runs it against ``learner_glue.device_learn``, alternating the
two in one run, on a ``PrioritizedReplayBank`` fed by live ``GpuVecEnv`` bins: the location network (selectedAction
500, 31 atoms) on BlockOut and general (irregular, R = 8) bins, and the order network (k = 10) on buffered BlockOut
bins.  GPU only.

    python tools/learn_bench.py [--bins 4096] [--reps 30] [--warmup 5] [--batch 64]

The trainer's arm is agent.py:68-125 in float32 torch on the port modules (``oracle/learn_port.py``, the reference's
forward and torch expressions), cudnn off, except for where the clouds come from: the reference gathers
``shapeArray[ids]`` on the host in each of its three forward passes, which is not timed here; ``DeviceShapeClouds``
gathers the same clouds on the device instead.  The device arm is ``device_learn``: the same gradient pass, the online
argmax through ``DeviceActor.act`` / ``DeviceOrderActor.act`` and the target through ``.target``.  Both arms share the
bank, start from the same weights and step their own copies.  A third arm, ``device_grad``, is
``device_learn(..., gradient="device")``: the device arm with the gradient pass through ``DeviceActor.log_prob``
(the candidate-row network and its backward as kernels) or ``DeviceOrderActor.log_prob`` (the order network's
per-slot layers, graph attention and heads and their backward as kernels).  The ``*_enc`` arms repeat
``device_grad`` (both levels) and ``device`` (order) with ``DeviceHeightEncoder`` swapped into the online net, so the
height encoder and its backward pass run as kernels too.  ``--levels order`` runs the order workload only.

Prints one JSON line per workload: ms per call and per part (sample, gradient pass, target = online argmax + target
pass + projection, step = loss + backward + clip + Adam, priority update) from CUDA events, medians and minima over
``--reps`` calls after ``--warmup``; the fraction of samples whose a* agrees between the two arms (the torch argmax
evaluated on the device arm's batches with the device arm's point indices); the card's name and power limit read in
the same run.

Before those, one JSON line per batch size for the height encoder alone (``bench: height_encoder``): the forward pass at
B = 4096 (an act over 4096 bins) and forward + backward at B = 64 and 512, ``DeviceHeightEncoder`` against torch
float32 (TF32 off) with cudnn off, as the reference trains, and with cudnn on; median and minimum ms per call from
CUDA events.  ``--encoder-only`` prints only these lines.

``--profile DIR`` instead profiles one arm (``--profile-arm``, default the order level's ``device_grad_enc``) in a run of
its own: ``torch.profiler`` with CUDA activities over ``--reps`` learns after ``--warmup``, one JSON line with the CUDA
time per call of the gradient pass's kernels and of the whole learn, grouped by kernel name, and the trace under DIR."""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from irbpp_b200 import shapes
from irbpp_b200.actor import DeviceActor, DeviceOrderActor
from irbpp_b200.height_encoder import DeviceHeightEncoder
from irbpp_b200.learner_glue import PrioritizedReplayBank, get_mask_from_state
from irbpp_b200.pointnet import DeviceShapeClouds
from irbpp_b200.vec_env import GpuVecEnv
from oracle.dqn_port import DQNPort
from oracle.learn_port import ReferenceDQN, ReferenceOrderDQN, distribution, torch_projection
from tools.act_bench import card

SEL, K, ATOMS = 500, 10, 31
V_MIN, V_MAX, GAMMA, N_STEP, NORM_CLIP, LR, ADAM_EPS = -1.0, 8.0, 0.99, 3, 10.0, 6.25e-5, 1.5e-4
PARTS = ("sample", "grad_pass", "target", "step", "priorities")


def filled_bank(lib, n, steps, seed, level, dev):
    k = K if level == "order" else 1
    env = GpuVecEnv(lib, None, num_envs=n, device=dev, buffer_size=k, item_seed=seed)
    state = env.reset().clone()
    bank = PrioritizedReplayBank(n, steps + 4, state.shape[1], dev, discount=GAMMA, multi_step=N_STEP, seed=seed,
                                 max_attempts=4096)
    gen = torch.Generator(device=dev); gen.manual_seed(seed)
    for _ in range(steps):
        if level == "order":
            action = torch.randint(0, k, (n,), device=dev, generator=gen)
            loc = env.get_action_candidates(action, as_tensor=True)
        else:
            loc = state
        q = torch.rand((n, SEL), device=dev, generator=gen)
        q[get_mask_from_state(loc, SEL) != 1] = -1.0
        if level != "order":
            action = q.argmax(1)
        nxt = env.step(q.argmax(1))[0]
        bank.append_from_env(env, state, action)
        state = nxt.clone()
    env.close()
    return bank


class Arm(object):
    """One learner: online / target port modules, Adam, and (device arm) the two device actors."""

    def __init__(self, online, target, clouds, support, device_arm, level, device_grad=False, device_encoder=False):
        if device_encoder:
            online.heightEncoder = DeviceHeightEncoder(online.heightEncoder)
        self.online, self.target, self.clouds, self.support, self.level = online, target, clouds, support, level
        self.opt = torch.optim.Adam(online.parameters(), lr=LR, eps=ADAM_EPS)
        self.device_arm, self.device_grad = device_arm, device_grad
        if device_arm:
            A = DeviceOrderActor if level == "order" else DeviceActor
            self.on_actor, self.tg_actor = A(online, clouds, support), A(target, clouds, support)
        self.agree = []

    def torch_argmax(self, next_states, counter):
        with torch.no_grad():
            src = torch.arange(self.clouds.S, dtype=torch.int32, device=next_states.device) if self.level == "order" \
                else next_states
            sf = self.online.shape_feature(self.clouds.sample(src, counter=counter))
            return (distribution(self.online, next_states, sf) * self.support).sum(2).argmax(1)

    def learn(self, bank, batch, ev):
        """One learn, with an event after each part (ev: six events)."""
        ev[0].record()
        idxs, states, actions, returns, next_states, nonterminals, weights, mem_ids = bank.sample(batch)
        B = states.shape[0]
        ev[1].record()
        if self.device_grad:
            log_ps_a = self.on_actor.log_prob(states, actions)
        else:
            log_ps = self.online(states, log=True)
            log_ps_a = log_ps[torch.arange(B, device=states.device), actions]
        ev[2].record()
        gn = GAMMA ** N_STEP
        with torch.no_grad():
            if self.device_arm:
                c = self.clouds.counter
                a = self.on_actor.act(next_states)
                self.target.reset_noise()
                m, _ = self.tg_actor.target(next_states, a, returns, nonterminals, V_MIN, V_MAX, gn, with_p=False)
            else:
                a = (self.online(next_states) * self.support).sum(2).argmax(1)
                self.target.reset_noise()
                pns_a = self.target(next_states)[torch.arange(B, device=states.device), a]
                m = torch_projection(pns_a, returns, nonterminals, self.support, V_MIN, V_MAX, gn)
        ev[3].record()
        loss = -torch.sum(m * log_ps_a, 1)
        self.online.zero_grad()
        (weights * loss).mean().backward()
        torch.nn.utils.clip_grad_norm_(self.online.parameters(), NORM_CLIP)
        self.opt.step()
        ev[4].record()
        bank.update_priorities(idxs, mem_ids, loss.detach())
        ev[5].record()
        torch.cuda.synchronize()
        if self.device_arm:                                   # outside the timed region
            self.agree.append(float((self.torch_argmax(next_states, c) == a).float().mean()))
        return [ev[i].elapsed_time(ev[i + 1]) for i in range(5)]


def run(name, level, lib, a, dev):
    torch.manual_seed(0)
    bank = filled_bank(lib, a.bins, 12, 3, level, dev)
    cloud_arr = np.random.default_rng(0).random((lib.num_shapes, 10000, 3)).astype(np.float32) * 0.1
    clouds = DeviceShapeClouds(cloud_arr, device=dev, item_col=K if level == "order" else SEL * 5)
    cls, kw = (ReferenceOrderDQN, dict(buffer_size=K)) if level == "order" else (ReferenceDQN, dict(selected_action=SEL))
    online = cls(clouds, atoms=ATOMS, **kw).to(dev).train()
    target = copy.deepcopy(online)
    for p in target.parameters():
        p.requires_grad = False
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=dev)
    arms = {"torch": Arm(online, target, clouds, support, False, level),
            "device": Arm(copy.deepcopy(online), copy.deepcopy(target), clouds, support, True, level)}
    if level == "order":
        arms["device_enc"] = Arm(copy.deepcopy(online), copy.deepcopy(target), clouds, support, True, level, False,
                                 True)
    arms["device_grad"] = Arm(copy.deepcopy(online), copy.deepcopy(target), clouds, support, True, level, True)
    arms["device_grad_enc"] = Arm(copy.deepcopy(online), copy.deepcopy(target), clouds, support, True, level, True,
                                  True)
    if a.profile:
        return profile(name, arms[a.profile_arm], bank, a)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    times = {n: [] for n in arms}
    for i in range(a.warmup + a.reps):
        for n, arm in arms.items():                           # alternate the two arms
            t = arm.learn(bank, a.batch, ev)
            if i >= a.warmup:
                times[n].append(t)
    out = {"workload": name, "level": level, "bins": a.bins, "batch": a.batch, "atoms": ATOMS,
           "k" if level == "order" else "selected_action": K if level == "order" else SEL, "reps": a.reps}
    for n, ts in times.items():
        ts = np.array(ts)
        tot = ts.sum(1)
        out[n] = {"ms_median": float(np.median(tot)), "ms_min": float(tot.min()),
                  "parts_ms_median": {p: float(np.median(ts[:, j])) for j, p in enumerate(PARTS)}}
    out["a_star_agreement"] = float(np.mean(arms["device"].agree))
    for n, ts in times.items():
        out[n]["ms_min_parts"] = {p: float(ts_p) for p, ts_p in zip(PARTS, np.array(ts).min(0))}
    out["grad_pass_share_of_device_learn"] = out["device"]["parts_ms_median"]["grad_pass"] / out["device"]["ms_median"]
    out["card"] = card()
    print(json.dumps(out))


def profile(name, arm, bank, a):
    """CUDA time per learn by kernel name, from torch.profiler (a run of its own: tracing slows the host)."""
    from torch.profiler import ProfilerActivity, profile as torch_profile
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    for _ in range(a.warmup):
        arm.learn(bank, a.batch, ev)
    os.makedirs(a.profile, exist_ok=True)
    with torch_profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            arm.learn(bank, a.batch, ev)
    prof.export_chrome_trace(os.path.join(a.profile, "learn_%s_%s.pt.trace.json" % (name, a.profile_arm)))
    rows = []
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        if us > 0 and e.device_type == torch.autograd.DeviceType.CUDA:
            rows.append((e.key, e.count / a.reps, us / 1000.0 / a.reps))
    rows.sort(key=lambda r: -r[2])
    out = {"profile": name, "arm": a.profile_arm, "batch": a.batch, "reps": a.reps,
           "cuda_ms_per_learn": sum(r[2] for r in rows), "launches_per_learn": sum(r[1] for r in rows),
           "kernels": [{"name": k[:90], "per_learn": c, "ms_per_learn": ms} for k, c, ms in rows[:40]],
           "card": card()}
    print(json.dumps(out))


def time_calls(fn, reps, warmup):
    """median and minimum ms of ``fn()`` over ``reps`` calls after ``warmup``, CUDA events around each call"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ts = []
    for i in range(warmup + reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        if i >= warmup:
            ts.append(ev[0].elapsed_time(ev[1]))
    return {"ms_median": float(np.median(ts)), "ms_min": float(np.min(ts))}


def encoder_bench(a, dev):
    """The height encoder alone: heightmaps read in place from observation rows of the location level's width."""
    torch.manual_seed(0)
    seq = DQNPort(selected_action=SEL, atoms=ATOMS).heightEncoder.to(dev)
    arms = {"device": DeviceHeightEncoder(copy.deepcopy(seq)), "torch": seq}
    for B, backward in ((4096, False), (64, True), (512, True)):
        rows = torch.rand((B, SEL * 5 + 9 + 1024), device=dev) * 0.3
        hm = rows[:, SEL * 5 + 9:].reshape(B, 1, 32, 32)
        g = torch.randn((B, 4, 8, 8), device=dev)
        out = {"bench": "height_encoder", "batch": B, "pass": "forward+backward" if backward else "forward",
               "reps": a.reps}

        def call(enc):
            if backward:
                for p in enc.parameters():
                    p.grad = None
                enc(hm).backward(g)
            else:
                with torch.no_grad():
                    enc(hm)
        for name, enc, cudnn in (("device", arms["device"], False), ("torch_cudnn_off", arms["torch"], False),
                                 ("torch_cudnn_on", arms["torch"], True)):
            with torch.backends.cudnn.flags(enabled=cudnn, allow_tf32=False):
                out[name] = time_calls(lambda: call(enc), a.reps, a.warmup)
        for name in ("torch_cudnn_off", "torch_cudnn_on"):
            out["speedup_vs_" + name] = out[name]["ms_median"] / out["device"]["ms_median"]
        out["card"] = card()
        print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bins", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--encoder-only", action="store_true")
    ap.add_argument("--levels", default="location,order")
    ap.add_argument("--profile", default=None, help="profile one arm instead, trace under this directory")
    ap.add_argument("--profile-arm", default="device_grad_enc")
    a = ap.parse_args()
    torch.backends.cudnn.enabled = False
    dev = torch.device("cuda:0")
    levels = a.levels.split(",")
    if a.profile:
        levels = ["order"]
    elif "location" in levels:
        encoder_bench(a, dev)
    if a.encoder_only:
        return
    if "location" in levels:
        run("blockout", "location", shapes.make_blockout_library(32, seed=1), a, dev)
        run("general", "location", shapes.make_irregular_library(16, seed=2, num_rotations=8), a, dev)
    if "order" in levels:
        run("blockout_buffered", "order", shapes.make_blockout_library(32, seed=1), a, dev)


if __name__ == "__main__":
    main()
