"""Step time of the 32 x 32 action grid (resolutionA = resolutionH = 0.01, stepSize 1) at 4096 bins on one GPU.

    python tools/fine_grid_bench.py [--steps 50] [--warmup 10] [--out result.json]

Method of bench.py: the device-resident loop (GpuVecEnv.step_device) with bench.py's random-valid device policy,
bench.BURN_IN + warm-up untimed steps so that the bins are spread over all episode phases, a 256 MiB L2 flush between
steps outside the timed interval, CUDA events around each step's library work; the median over the steps is reported.
Workloads: Cube boxes at R = 2 and BlockOut-like polycubes at R = 4, each on the fine grid and, as the reference point of
the same run, on the 16 x 16 grid (resolutionA 0.02).  The card's name and power limit are read in the same run and
printed with the figures: a number is only meaningful with what it was measured on.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the device policy and the burn-in length of the flagship benchmark)

WORKLOADS = [("cube_fine_R2", "cube", 2, 0.01), ("blockout_fine_R4", "blockout", 4, 0.01),
             ("cube_R2", "cube", 2, 0.02), ("blockout_R4", "blockout", 4, 0.02)]


def card_info(index):
    """Name, power limit and max SM clock of the card, read with nvidia-smi's query interface (read only)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:                                  # noqa: BLE001  (the figures are still printed)
        return {"name": None, "error": "nvidia-smi: %s" % e}


def time_workload(torch, dev, shape, R, res_act, bins, steps, warmup, flush, gen):
    from irbpp_b200 import shapes
    from irbpp_b200.vec_env import GpuVecEnv
    if shape == "cube":
        lib = shapes.make_cube_library(seed=3, num_rotations=R, resolutionAct=res_act)
    else:
        lib = shapes.make_blockout_library(32, seed=1, num_rotations=R, resolutionAct=res_act)
    seqs = shapes.make_sequences(bins, bench.SEQ_LEN, lib.num_shapes, seed=0)
    env = GpuVecEnv(lib, seqs, device=dev, selected_action=bench.SEL)
    obs = env.reset()
    for _ in range(bench.BURN_IN + warmup):
        obs, _ = env.step_device(bench.device_policy(torch, obs, gen))
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize(dev)
    for i in range(steps):
        acts = bench.device_policy(torch, obs, gen)
        flush.fill_(float(i))                               # L2 flush, outside the event pair
        ev[i][0].record()
        obs, _ = env.step_device(acts)
        ev[i][1].record()
    torch.cuda.synchronize(dev)
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    env.close()
    return {"ms_per_step_median": float(np.median(ms)), "ms_per_step_min": float(ms.min()),
            "ms_per_step_max": float(ms.max()), "steps": steps, "bins": bins, "R": R, "resolutionA": res_act,
            "Ax": env.Ax, "Ay": env.Ay}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--bins", type=int, default=4096)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("fine_grid_bench.py: no CUDA device; the library has no CPU path")
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev)
    gen.manual_seed(1234)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    import gc
    gc.collect()
    gc.disable()
    result = {"card": card_info(0), "torch_device_name": torch.cuda.get_device_name(dev), "workloads": {}}
    for name, shape, R, res in WORKLOADS:
        result["workloads"][name] = time_workload(torch, dev, shape, R, res, args.bins, args.steps, args.warmup, flush, gen)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
