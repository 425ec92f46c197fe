#!/usr/bin/env python
"""Time Agent.act at N bins: the location network in torch float32 as trainer.py runs it (cudnn disabled, the
shape encoder on the sampled clouds of every bin) against DeviceShapeClouds.features + DeviceActor.act
(csrc/irbpp_actor.cuh), alternating the two in one run, on the BlockOut and the general (irregular, R = 8) workloads
after a burn-in of random valid steps.  GPU only.

    python tools/act_bench.py [--bins 4096] [--reps 20] [--warmup 3]

prints one JSON line per workload: ms per act of both paths (CUDA events), the valid rows, achieved FLOP/s from the
layer shapes, the cost of rebuilding the NoisyLinear weights, the agreement of the two paths' actions, and the card's
name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from irbpp_b200 import shapes
from irbpp_b200.actor import DeviceActor
from irbpp_b200.learner_glue import get_mask_from_state
from irbpp_b200.pointnet import DeviceShapeClouds
from irbpp_b200.vec_env import GpuVecEnv
from oracle.dqn_port import DQNPort

SEL = 500
# multiply-adds from the layer shapes (DESIGN.md section 4)
MAC_ROW_TORCH = 4 * 32 + 32 * 128 + 512 * 256 + 256 * 128 + 128 * 128 + 128 * 31           # 188 416
MAC_BIN_TORCH = 65536 + 524288 + 73728 + 128 * 128 + 128 * 31                             # convs + value head
MAC_ROW_FUSED = 4 * 32 + 32 * 128 + 128 * 256 + 256 * 128 + 128 * 128 + 128 * 31          # 90 112
MAC_BIN_FUSED = 65536 + 524288 + 73728 + 384 * 256 + 128 * 128 + 128 * 31                 # 782 208
MAC_ENCODER_POINT = 3 * 128 + 128 * 128


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                      # noqa: BLE001
        out = "nvidia-smi unavailable: %s" % e
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": out}


def burn_in(lib, n, steps, seed, dev):
    env = GpuVecEnv(lib, None, num_envs=n, device=dev, item_seed=seed)
    state = env.reset()
    gen = torch.Generator(device=dev); gen.manual_seed(seed)
    for _ in range(steps):
        q = torch.rand((n, SEL), device=dev, generator=gen)
        q[get_mask_from_state(state, SEL) != 1] = -1.0
        state = env.step(q.argmax(1))[0]
    state = state.clone()
    env.close()
    return state


def events_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps, out


def run(name, lib, a, dev):
    torch.manual_seed(0)
    state = burn_in(lib, a.bins, 12, 3, dev)
    mask = get_mask_from_state(state, SEL)
    n_valid = int((mask == 1).sum())
    net = DQNPort().to(dev).train()
    support = torch.linspace(-10, 10, 31, device=dev)
    cloud_arr = np.random.default_rng(0).random((lib.num_shapes, 10000, 3)).astype(np.float32) * 0.1
    clouds = DeviceShapeClouds(cloud_arr, device=dev)
    actor = DeviceActor(net, clouds, support)

    def torch_act():                            # agent.py:51-58 on model.py's forward, float32
        with torch.no_grad():
            sf = net.shape_feature(clouds.sample(state))
            return net.act(state, sf, support, mask)

    def fused_act():
        return actor.act(state, mask)

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
    t_rebuild, _ = events_ms(actor.effective_weights, 50)
    agree = float((a_torch == a_fused).float().mean())
    ms_torch, ms_fused = float(np.median(t_torch)), float(np.median(t_fused))
    flop_torch = 2.0 * (a.bins * SEL * MAC_ROW_TORCH + a.bins * MAC_BIN_TORCH + a.bins * 1024 * MAC_ENCODER_POINT)
    flop_fused = 2.0 * (n_valid * MAC_ROW_FUSED + a.bins * MAC_BIN_FUSED) + 2.0 * lib.num_shapes * 1024 * MAC_ENCODER_POINT
    return {"workload": name, "bins": a.bins, "selected_action": SEL, "valid_rows": n_valid,
            "valid_rows_per_bin": n_valid / a.bins, "reps": a.reps,
            "torch_fp32_ms": ms_torch, "torch_fp32_ms_min": float(np.min(t_torch)),
            "fused_ms": ms_fused, "fused_ms_min": float(np.min(t_fused)), "speedup": ms_torch / ms_fused,
            "torch_tflops": flop_torch / ms_torch / 1e9, "fused_tflops_counted": flop_fused / ms_fused / 1e9,
            "fused_flop_counted": flop_fused, "weight_rebuild_ms": t_rebuild,
            "actions_equal_fraction": agree, "cudnn": torch.backends.cudnn.enabled}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bins", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("act_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    for name, lib in (("blockout", shapes.make_blockout_library(32, seed=1)),
                      ("general", shapes.make_irregular_library(32, seed=2, num_rotations=8))):
        out = run(name, lib, a, dev)
        out.update(info)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
