#!/usr/bin/env python
"""Device time per batched step of one library build on several workloads (GPU only, no CPU arm).

    IRBPP_LIB=irbpp_b200/lib/libirbpp_x.so python tools/kbench.py [--workloads blockout,irregular8,...] [--e2e]

One JSON line per workload: per-step CUDA-event time (L2 flushed between steps, outside the events), the
torch stand-in policy is NOT inside the events.  Used to compare two builds of the library (IRBPP_LIB)."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from irbpp_b200 import shapes
from irbpp_b200.vec_env import GpuVecEnv

SEL = 500


def make(name):
    if name == "blockout":
        return shapes.make_blockout_library(32, seed=1, num_rotations=4), 1
    if name == "cube":
        return shapes.make_cube_library(seed=3), 1
    if name == "irregular8":
        return shapes.make_irregular_library(32, seed=2, num_rotations=8), 1
    if name == "irregular24":
        return shapes.make_irregular_library(32, seed=2, num_rotations=24), 1
    if name == "buffered10":
        return shapes.make_blockout_library(32, seed=1, num_rotations=4), 10
    raise SystemExit("unknown workload " + name)


def policy(obs, gen):
    n = obs.shape[0]
    mask = obs[:, :SEL * 5].view(n, SEL, 5)[:, :, 4] == 1
    return torch.argmax(torch.rand((n, SEL), device=obs.device, generator=gen) + mask.float(), dim=1)


def run(name, n, steps, burn, e2e):
    lib, k = make(name)
    seqs = shapes.make_sequences(n, 128, lib.num_shapes, seed=0)
    env = GpuVecEnv(lib, seqs, device="cuda:0", buffer_size=k)
    gen = torch.Generator(device="cuda:0"); gen.manual_seed(1)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda:0")
    obs = env.reset()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]

    def one(timed=None):
        nonlocal obs
        if k > 1:
            order = torch.randint(0, k, (n,), device="cuda:0", generator=gen)
            if timed is not None:
                flush.fill_(1.0); timed[0].record()
            loc = env.get_action_candidates(order, as_tensor=True)
            acts = policy(loc, gen)
            obs, _ = env.step_device(acts)
            if timed is not None:
                timed[1].record()
        else:
            acts = policy(obs, gen)
            if timed is not None:
                flush.fill_(1.0); timed[0].record()
            obs, _ = env.step_device(acts)
            if timed is not None:
                timed[1].record()
    for _ in range(burn):
        one()
    torch.cuda.synchronize()
    for s in range(steps):
        one(ev[s])
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    out = {"workload": name, "bins": n, "R": lib.num_rotations, "k": k, "ms_per_step": round(float(np.mean(ms)), 5),
           "ms_min": round(float(np.min(ms)), 5), "ms_p90": round(float(np.percentile(ms, 90)), 5),
           "lib": os.path.basename(os.environ.get("IRBPP_LIB", "libirbpp.so"))}
    if e2e and k == 1:
        t = 0.0
        for s in range(steps):
            acts = policy(obs, gen).cpu().numpy()
            flush.fill_(1.0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            obs, rew, done, infos = env.step(acts)
            torch.cuda.synchronize()
            t += time.perf_counter() - t0
        out["e2e_ms"] = round(1e3 * t / steps, 5)
    print(json.dumps(out), flush=True)
    env.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="blockout,irregular8")
    ap.add_argument("--bins", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--burn", type=int, default=150)
    ap.add_argument("--e2e", action="store_true")
    a = ap.parse_args()
    for w in a.workloads.split(","):
        run(w, a.bins, a.steps, a.burn, a.e2e)


if __name__ == "__main__":
    main()
