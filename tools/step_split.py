#!/usr/bin/env python
"""Device time of each kernel of a step on bench.py's workload, from torch.profiler in a run of its own.  GPU only.

    python tools/step_split.py [--config blockout] [--steps 50] [--out DIR]

Same library, sequences, policy, burn-in and L2 flush between steps as ``bench.py --config CONFIG`` (k = 1 configs).
Prints one JSON object: ms per step of every kernel the steps launched (the library's and the stand-in policy's; the
flush runs outside the profiled window), the scan kernel's share of the two step kernels, and the card's name and power
limit.  ``IRBPP_LIB`` selects the library build, as for bench.py.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from irbpp_b200 import shapes  # noqa: E402
from irbpp_b200.vec_env import GpuVecEnv  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().split(",")] if q.returncode == 0 else (torch.cuda.get_device_name(0), "?", "?")
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="blockout", choices=[c for c, s in bench.CONFIGS.items() if s["k"] == 1])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", help="also write the result as DIR/step_split_<config>.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_split.py: no CUDA device")
    spec = bench.CONFIGS[args.config]
    n = spec["bins"]
    dev = torch.device("cuda", 0)
    lib = bench.make_library(args.config)
    seqs = shapes.make_sequences(n, bench.SEQ_LEN, lib.num_shapes, seed=0)
    env = GpuVecEnv(lib, seqs, device=dev, selected_action=bench.SEL, buffer_size=1)
    gen = torch.Generator(device=dev)
    gen.manual_seed(1234)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    obs = env.reset()
    for _ in range(bench.BURN_IN + args.warmup):
        obs, _ = env.step_device(bench.device_policy(torch, obs, gen))
    torch.cuda.synchronize(dev)

    from torch.profiler import ProfilerActivity, profile
    totals = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            choice = bench.device_policy(torch, obs, gen)
            flush.fill_(float(i))                       # L2 flush between steps, as bench.py does
            obs, _ = env.step_device(choice)
        torch.cuda.synchronize(dev)
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0.0)
        if t > 0 and "fill" not in ev.key.lower():
            totals[ev.key] = totals.get(ev.key, 0.0) + t
    ms = {k: round(v / 1e3 / args.steps, 4) for k, v in sorted(totals.items(), key=lambda kv: -kv[1])}
    scan = sum(v for k, v in ms.items() if "irbpp_scan" in k)
    cand = sum(v for k, v in ms.items() if "irbpp_candidates" in k)
    out = {"config": args.config, "bins": n, "steps": args.steps, "lib": os.environ.get("IRBPP_LIB", "default"),
           "card": card(), "kernel_ms_per_step": ms, "scan_ms": round(scan, 4), "candidates_ms": round(cand, 4),
           "scan_share_of_step_kernels": round(scan / (scan + cand), 3) if scan + cand > 0 else None}
    env.close()
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_split_%s.json" % args.config), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
