#!/usr/bin/env python
"""Time the order network's act at N bins, k = 10 (the buffered configuration): the order network in torch float32
against DeviceShapeClouds.features + DeviceOrderActor.act (csrc/irbpp_order_actor.cuh), alternating the two in one
run, on the BlockOut and the general (irregular, R = 8) workloads after a burn-in of random hierarchical steps; then
one whole hierarchical actor-loop iteration on the device (order act, get_action_candidates, location act, step).
GPU only.

    python tools/order_act_bench.py [--bins 4096] [--reps 20] [--warmup 3] [--iters 30]

The torch arm is model.py:355-404 as written except for where the slots' clouds come from: the reference gathers
shapeArray[ids] for all N * k slots on the host (about 4.9 GB per act at N = 4096, k = 10), which is not timed here;
DeviceShapeClouds.sample gathers the same [N * k, 1024, 3] clouds on the device instead, in chunks of 512 bins so that
the shape encoder's intermediates fit, and the shape encoder then runs on every slot's cloud as in the reference.

Prints one JSON line per workload (ms per act of both paths from CUDA events, medians and minima, the agreement of
their actions) and one for the loop (ms per iteration and per part, medians), each with the card's name and power
limit read in the same run."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from irbpp_b200 import shapes
from irbpp_b200.actor import DeviceActor, DeviceOrderActor
from irbpp_b200.learner_glue import get_mask_from_state
from irbpp_b200.pointnet import DeviceShapeClouds
from irbpp_b200.vec_env import GpuVecEnv
from oracle.dqn_port import DQNPort
from oracle.order_dqn_port import OrderDQNPort
from tools.act_bench import card, events_ms

SEL, K, CHUNK = 500, 10, 512


def burn_in(lib, n, steps, seed, dev):
    env = GpuVecEnv(lib, None, num_envs=n, device=dev, buffer_size=K, item_seed=seed)
    state = env.reset()
    gen = torch.Generator(device=dev); gen.manual_seed(seed)
    for _ in range(steps):
        loc = env.get_action_candidates(torch.randint(0, K, (n,), device=dev, generator=gen), as_tensor=True)
        q = torch.rand((n, SEL), device=dev, generator=gen)
        q[get_mask_from_state(loc, SEL) != 1] = -1.0
        state = env.step(q.argmax(1))[0]
    return env, state.clone()


def run(name, lib, a, dev):
    torch.manual_seed(0)
    env, state = burn_in(lib, a.bins, 12, 3, dev)
    env.close()
    net = OrderDQNPort(buffer_size=K).to(dev).train()
    support = torch.linspace(-10, 10, 31, device=dev)
    cloud_arr = np.random.default_rng(0).random((lib.num_shapes, 10000, 3)).astype(np.float32) * 0.1
    clouds = DeviceShapeClouds(cloud_arr, device=dev)
    actor = DeviceOrderActor(net, clouds, support)
    slot_ids = torch.arange(CHUNK * K, device=dev, dtype=torch.float32).reshape(CHUNK, K)

    def torch_act():                            # agent.py:51-58 on model.py:355-404, float32, shape encoder per slot,
        # on the index set the next fused act draws (counter), so that both arms of a rep see the same points
        out = []
        with torch.no_grad():
            for i in range(0, a.bins, CHUNK):
                obs = state[i:i + CHUNK]
                ids = obs[:, :K].long().reshape(-1).to(torch.int32)
                feat = net.shape_feature(clouds.sample(ids, counter=clouds.counter))     # [chunk * K, 128]
                obs = torch.cat((slot_ids[:obs.shape[0]], obs[:, K:]), dim=1)           # slot j of bin b -> row b*K+j
                out.append(net.act(obs, feat, support))
        return torch.cat(out)

    def fused_act():
        return actor.act(state)

    torch.backends.cudnn.enabled = False        # trainer.py: enable_cudnn defaults off
    for _ in range(a.warmup):
        torch_act(); fused_act()
    torch.cuda.synchronize()
    t_torch, t_fused = [], []
    for _ in range(a.reps):                     # alternating
        t, a_torch = events_ms(torch_act, 1)
        t_torch.append(t)
        t, a_fused = events_ms(fused_act, 1)
        t_fused.append(t)
    ms_torch, ms_fused = float(np.median(t_torch)), float(np.median(t_fused))
    return {"workload": name, "bins": a.bins, "buffer_size": K, "shapes": lib.num_shapes, "reps": a.reps,
            "torch_fp32_ms": ms_torch, "torch_fp32_ms_min": float(np.min(t_torch)),
            "fused_ms": ms_fused, "fused_ms_min": float(np.min(t_fused)), "speedup": ms_torch / ms_fused,
            "actions_equal_fraction": float((a_torch == a_fused).float().mean()), "cudnn": torch.backends.cudnn.enabled}


def loop(a, dev):
    """One hierarchical actor-loop iteration (trainer.py:261-281) with both device actors, ms per part (host clock
    around device-synchronised parts) and per iteration (no synchronisation inside)."""
    torch.manual_seed(0)
    lib = shapes.make_blockout_library(32, seed=1)
    cloud_arr = np.random.default_rng(0).random((lib.num_shapes, 10000, 3)).astype(np.float32) * 0.1
    clouds = DeviceShapeClouds(cloud_arr, device=dev, item_col=SEL * 5)
    support = torch.linspace(-10, 10, 31, device=dev)
    order_actor = DeviceOrderActor(OrderDQNPort(buffer_size=K).to(dev).train(), clouds, support)
    loc_actor = DeviceActor(DQNPort().to(dev).train(), clouds, support)
    env, state = burn_in(lib, a.bins, 12, 3, dev)
    parts = {"order act": [], "get_action_candidates": [], "location act": [], "env.step": []}

    def lap(name, t):
        torch.cuda.synchronize()
        now = time.perf_counter()
        parts[name].append(1e3 * (now - t))
        return now

    def iteration(state):
        order = order_actor.act(state)
        loc = env.get_action_candidates(order, as_tensor=True)
        return env.step(loc_actor.act(loc, get_mask_from_state(loc, SEL)))[0]

    for _ in range(a.warmup):
        state = iteration(state)
    whole = []
    for _ in range(a.iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        state = iteration(state)
        torch.cuda.synchronize()
        whole.append(1e3 * (time.perf_counter() - t0))
    for _ in range(a.iters):
        torch.cuda.synchronize()
        t = time.perf_counter()
        order = order_actor.act(state)
        t = lap("order act", t)
        loc = env.get_action_candidates(order, as_tensor=True)
        t = lap("get_action_candidates", t)
        action = loc_actor.act(loc, get_mask_from_state(loc, SEL))
        t = lap("location act", t)
        state = env.step(action)[0]
        lap("env.step", t)
    env.close()
    return {"workload": "hierarchical loop, blockout", "bins": a.bins, "buffer_size": K, "iters": a.iters,
            "ms_per_iteration": float(np.median(whole)), "ms_per_iteration_min": float(np.min(whole)),
            "ms_per_part_synchronised": {k: round(float(np.median(v)), 4) for k, v in parts.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bins", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("order_act_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    for name, lib in (("blockout", shapes.make_blockout_library(32, seed=1)),
                      ("general", shapes.make_irregular_library(32, seed=2, num_rotations=8))):
        out = run(name, lib, a, dev)
        out.update(info)
        print(json.dumps(out), flush=True)
    out = loop(a, dev)
    out.update(info)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
