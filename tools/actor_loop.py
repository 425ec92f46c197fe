#!/usr/bin/env python
"""The reference's actor loop (trainer.py:157-186: mask -> act -> envs.step -> infos -> replay append [-> sample])
at N = 4096 on one GPU, in two forms: the loop as trainer.py writes it (per-bin Python loops over infos and over N
replay memories) and the same loop through irbpp_b200.learner_glue (batched).  The agent is a stand-in with the
reference's interface (act(state, mask) -> greedy masked argmax of a random Q map).  GPU only.

    python tools/actor_loop.py [--iters 30] [--bins 4096] [--skip-reference-style]
prints one JSON line: iterations/s and env-steps/s of both forms next to the env-only e2e step time."""
import argparse, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from irbpp_b200 import shapes, learner_glue as glue
from irbpp_b200.vec_env import GpuVecEnv

SEL = 500


class StandInAgent(object):
    """Agent.act (agent.py:47-58): argmax over actions of a Q map with masked-out actions at -inf."""

    def __init__(self, device, seed=0):
        self.gen = torch.Generator(device=device); self.gen.manual_seed(seed)

    def act(self, state, mask):
        q = torch.rand(mask.shape, device=state.device, generator=self.gen)
        q[(1 - mask).bool()] = -float("inf")
        return q.argmax(1)


def count_kernels(fn):
    """Kernels (not copies or memsets) that one call of fn puts on the GPU, from torch.profiler's CUDA events."""
    from torch.profiler import profile, ProfilerActivity
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(); torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--bins", type=int, default=4096)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--replay-frequency", type=int, default=4)
    ap.add_argument("--capacity", type=int, default=64, help="transitions per environment in the replay bank")
    ap.add_argument("--skip-reference-style", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = shapes.make_blockout_library(32, seed=1)
    n = a.bins
    env = GpuVecEnv(lib, None, num_envs=n, device=dev, item_seed=1)
    agent = StandInAgent(dev)
    reward_clip = torch.ones((n, 1)) * 10.0
    out = {"bins": n, "iters": a.iters}

    def warm(state, k=20):
        for _ in range(k):
            state = env.step(agent.act(state, glue.get_mask_from_state(state, SEL)).cpu().numpy())[0]
        return state

    # ---- env only (what bench.py's e2e times) ----
    state = warm(env.reset(), 60)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(a.iters):
        action = agent.act(state, glue.get_mask_from_state(state, SEL))
        state, reward, done, infos = env.step(action.cpu().numpy())
    torch.cuda.synchronize(); dt = time.perf_counter() - t0
    out["act_plus_env_step_only"] = {"iters_per_s": a.iters / dt, "env_steps_per_s": n * a.iters / dt}

    # ---- the loop through learner_glue (batched) ----
    bank = glue.ReplayBank(n, a.capacity, env.obs_len, dev)
    stats = glue.EpisodeStats()
    parts = {"mask+act": 0.0, "env.step": 0.0, "episode stats": 0.0, "replay append": 0.0, "replay sample": 0.0}

    def lap(name, t):
        torch.cuda.synchronize()
        now = time.perf_counter()
        parts[name] += now - t
        return now
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for T in range(1, a.iters + 1):
        t = time.perf_counter()
        mask = glue.get_mask_from_state(state, SEL)
        action = agent.act(state, mask)
        acts_host = action.cpu().numpy()
        t = lap("mask+act", t)
        next_state, reward, done, infos = env.step(acts_host)
        t = lap("env.step", t)
        stats.update(done, infos)
        t = lap("episode stats", t)
        bank.append_from_env(env, state, action, reward_clip=10.0)       # reward clip + append on the device
        t = lap("replay append", t)
        if T % a.replay_frequency == 0 and len(bank) >= 2:
            batch = bank.sample(a.batch_size)
            t = lap("replay sample", t)
        state = next_state
    torch.cuda.synchronize(); dt = time.perf_counter() - t0
    out["glue_loop"] = {"iters_per_s": a.iters / dt, "env_steps_per_s": n * a.iters / dt, "episodes": stats.episodes,
                        "mean_ratio_last10": float(np.mean(stats.episode_ratio)) if stats.episode_ratio else None,
                        "ms_per_iter_by_part": {k: round(1e3 * v / a.iters, 4) for k, v in parts.items()}}

    # ---- the prioritized bank (memory.py's replay, csrc/irbpp_replay.cuh) beside the uniform bank ----
    pbank = glue.PrioritizedReplayBank(n, a.capacity, env.obs_len, dev, seed=1)
    ubank = glue.ReplayBank(n, a.capacity, env.obs_len, dev)
    pparts = {"prioritized append": 0.0, "prioritized sample": 0.0, "prioritized update": 0.0,
              "uniform append": 0.0, "uniform sample": 0.0}
    parts = pparts
    rounds = 0
    for T in range(1, a.iters + 1):
        action = agent.act(state, glue.get_mask_from_state(state, SEL))
        next_state, reward, done, infos = env.step(action.cpu().numpy())
        torch.cuda.synchronize(); t = time.perf_counter()
        ubank.append_from_env(env, state, action, reward_clip=10.0)
        t = lap("uniform append", t)
        pbank.append_from_env(env, state, action, reward_clip=10.0)
        t = lap("prioritized append", t)
        if T >= a.capacity // 2:
            ubank.sample(a.batch_size)
            t = lap("uniform sample", t)
            batch = pbank.sample(a.batch_size)
            t = lap("prioritized sample", t)
            loss = torch.rand(batch[0].shape[0], device=dev)
            torch.cuda.synchronize(); t = time.perf_counter()
            pbank.update_priorities(batch[0], batch[7], loss)
            t = lap("prioritized update", t)
            rounds += 1
        state = next_state
    out["replay_banks"] = {"ms_per_call": {k: round(1e3 * v / (a.iters if "append" in k else max(rounds, 1)), 4)
                                           for k, v in pparts.items()},
                           "kernel_launches_per_call": {
                               "prioritized append": count_kernels(lambda: pbank.append_from_env(env, state, action)),
                               "prioritized sample": count_kernels(lambda: pbank.sample(a.batch_size)),
                               "prioritized update": count_kernels(lambda: pbank.update_priorities(batch[0], batch[7], loss)),
                               "uniform append": count_kernels(lambda: ubank.append_from_env(env, state, action)),
                               "uniform sample": count_kernels(lambda: ubank.sample(a.batch_size))},
                           "sample_rounds": rounds, "capacity": a.capacity, "batch_size": a.batch_size}

    # ---- the loop as trainer.py:157-186 writes it (per-bin Python) ----
    if not a.skip_reference_style:
        from collections import deque
        mem = [deque(maxlen=a.capacity) for _ in range(n)]
        episode_rewards, episode_ratio, episode_counter = deque(maxlen=10), deque(maxlen=10), deque(maxlen=10)
        iters = max(3, a.iters // 10)
        torch.cuda.synchronize(); t0 = time.perf_counter()
        for T in range(1, iters + 1):
            mask = glue.get_mask_from_state(state, SEL)
            action = agent.act(state, mask)
            next_state, reward, done, infos = env.step(action.cpu().numpy())
            validSample = []
            for _ in range(len(infos)):
                validSample.append(infos[_]['Valid'])
                if done[_] and infos[_]['Valid']:
                    episode_rewards.append(infos[_]['episode']['r'])
                    if 'ratio' in infos[_].keys():
                        episode_ratio.append(infos[_]['ratio'])
                    if 'counter' in infos[_].keys():
                        episode_counter.append(infos[_]['counter'])
            reward = torch.maximum(torch.minimum(reward, reward_clip), -reward_clip)
            for i in range(len(state)):
                if validSample[i]:
                    mem[i].append((state[i], action[i], reward[i], done[i]))
            state = next_state
        torch.cuda.synchronize(); dt = time.perf_counter() - t0
        out["reference_style_loop"] = {"iters_per_s": iters / dt, "env_steps_per_s": n * iters / dt, "iters": iters}
    print(json.dumps(out))
    env.close()


if __name__ == "__main__":
    main()
