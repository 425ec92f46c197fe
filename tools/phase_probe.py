#!/usr/bin/env python
"""Per-phase SM cycles of the two step kernels on the bench workload (steady state).  GPU only.

    python tools/phase_probe.py                       # phases + work counters of the candidates kernel

Thread 0 of every CTA adds clock64() differences to eight counters (include/irbpp.h,
irbpp_debug_phase_cycles); the numbers are cycles as seen by warp 0 of a CTA, barrier waits included.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from irbpp_b200 import shapes  # noqa: E402
from irbpp_b200.vec_env import GpuVecEnv  # noqa: E402

CONFIG = os.environ.get("IRBPP_PROBE_CONFIG", "blockout")       # any bench.py --config with k = 1
N_ENVS = bench.CONFIGS[CONFIG]["bins"]
lib = bench.make_library(CONFIG)
seqs = shapes.make_sequences(N_ENVS, bench.SEQ_LEN, lib.num_shapes, seed=0)
env = GpuVecEnv(lib, seqs, device="cuda:0")
gen = torch.Generator(device="cuda:0")
gen.manual_seed(1)
obs = env.reset()
for _ in range(bench.BURN_IN):
    obs, _ = env.step_device(bench.device_policy(torch, obs, gen))
env.debug_phase_cycles(True)
n = 20
for _ in range(n):
    obs, _ = env.step_device(bench.device_policy(torch, obs, gen))
c = env.debug_phase_cycles(False).astype(np.float64) / n
scan_ctas = N_ENVS
bins_per_cta = 8 if lib.num_rotations >= 8 else 4          # envs_per_cta_for(R), csrc/irbpp_kernels.cuh
cand_ctas = N_ENVS // bins_per_cta
out = {"lib": os.environ.get("IRBPP_LIB", "default"), "config": CONFIG, "bins_per_candidates_cta": bins_per_cta,
       "scan_kernel_cycles_per_cta": {"load + apply action (phase A)": round(c[0] / scan_ctas),
                                      "observation, pose scan, level bitmaps": round(c[1] / scan_ctas)},
       "candidates_kernel_cycles_per_cta": {"contour tasks (phase C)": round(c[2] / cand_ctas),
                                            "select / pad (phase D)": round(c[3] / cand_ctas)},
       "work_per_cta": {"level images": round(c[4] / cand_ctas, 1), "start-pixel tasks": round(c[5] / cand_ctas, 1),
                        "rounds": round(c[6] / cand_ctas, 2), "overflow redos (> 64 points)": round(c[7] / cand_ctas, 3)}}
print(json.dumps(out, indent=1))
