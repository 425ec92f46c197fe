#!/usr/bin/env python
"""Cost of the item sources on the GPU (prints JSON lines):

* ``step``: BlockOut step time (bench library, 4096 bins, device first-valid policy) with instance-grouped draws
  against the uniform generator, CUDA events over --steps steps, the two alternated --reps times;
* ``evaluate``: wall time of ``evaluation.evaluate`` over --trajs trajectories of --items BlockOut items with
  --eval-envs bins and the same device policy, against the serial ``SingleGpuEnv`` loop of ``tools.test`` over the
  first --serial of those trajectories.

    python tools/item_source_probe.py [--steps 200 --reps 3 --trajs 2000 --items 100 --eval-envs 2000 --serial 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def first_valid_torch(obs, sel=500):
    import torch
    valid = obs[:, :sel * 5].reshape(obs.shape[0], sel, 5)[:, :, 4] == 1
    return torch.argmax(valid.to(torch.int32), dim=1)


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "?"


def time_steps(env, steps, warmup):
    import torch
    obs = env.reset()
    for _ in range(warmup):
        obs, _, _, _ = env.step(first_valid_torch(obs))
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        obs, _, _, _ = env.step(first_valid_torch(obs))
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--trajs", type=int, default=2000)
    ap.add_argument("--items", type=int, default=100)
    ap.add_argument("--eval-envs", type=int, default=2000)
    ap.add_argument("--serial", type=int, default=20)
    args = ap.parse_args()
    import torch
    from irbpp_b200 import shapes
    from irbpp_b200.evaluation import evaluate
    from irbpp_b200.single_env import SingleGpuEnv
    from irbpp_b200.vec_env import GpuVecEnv
    lib = shapes.make_blockout_library(32, seed=1, num_rotations=4)
    groups = [list(range(g, 32, 8)) for g in range(8)]          # 8 groups of 4 shapes
    gpu = gpu_name()
    res = {"uniform": [], "instance_groups": []}
    for _ in range(args.reps):
        for mode in res:
            env = GpuVecEnv(lib, None, num_envs=4096, item_seed=3,
                            item_groups=groups if mode == "instance_groups" else None)
            res[mode].append(time_steps(env, args.steps, args.warmup))
            env.close()
    print(json.dumps({"probe": "step", "gpu": gpu, "bins": 4096, "steps": args.steps,
                      "ms_per_step": {k: [round(v, 4) for v in vs] for k, vs in res.items()}}))

    rng = np.random.default_rng(0)
    trajs = [[int(v) for v in rng.integers(0, lib.num_shapes, size=args.items)] for _ in range(args.trajs + 1)]
    evaluate(lib, trajs, first_valid_torch, args.eval_envs, first=1, count=64)           # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = evaluate(lib, trajs, first_valid_torch, args.eval_envs, first=1, count=args.trajs)
    torch.cuda.synchronize()
    t_batch = time.perf_counter() - t0
    env = SingleGpuEnv(lib, trajectories=trajs, first_trajectory=1)
    t0 = time.perf_counter()
    lengths = []
    for _ in range(args.serial):
        state, n = env.reset(), 0
        while True:
            v = np.nonzero(state[:2500].reshape(500, 5)[:, 4] == 1)[0]
            state, _, done, _ = env.step(int(v[0]) if len(v) else 0)
            n += 1
            if done:
                break
        lengths.append(n)
    t_serial = time.perf_counter() - t0
    env.close()
    assert lengths == list(out["length"][:args.serial])
    print(json.dumps({"probe": "evaluate", "gpu": gpu, "trajectories": args.trajs, "items": args.items,
                      "bins": args.eval_envs, "evaluate_s": round(t_batch, 3),
                      "mean_length": float(np.mean(out["length"])), "max_length": int(np.max(out["length"])),
                      "serial_trajectories": args.serial, "serial_s": round(t_serial, 3),
                      "serial_s_per_trajectory": round(t_serial / args.serial, 4),
                      "summary": out["summary"]}))


if __name__ == "__main__":
    main()
