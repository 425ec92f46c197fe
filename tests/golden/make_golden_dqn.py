"""Generate ``dqn_act.npz`` from the UNMODIFIED reference network (``model.py`` ``DQNBPP``, location level) and
``Agent.act`` (``agent.py:51-58``, restated in three lines below because ``Agent.__init__`` needs the whole trainer).

Run in the build container (needs the reference tree and torch):

    python tests/golden/make_golden_dqn.py

``model.py`` is executed from where it lies, after ``oracle/ref_loader.py`` has installed its import stand-ins
(``from tools import init``).  A seeded ``DQNBPP(args, 500, shapeArray)`` with the reference defaults (atoms 31,
hidden 128, noisy_std 0.5) runs on the CPU in float32 over 44 observations of the in-repo oracle environments:

* kind 0: BlockOut, 4 rotations, mid-episode (lowest-H policy);
* kind 1: irregular shapes, 24 rotations, with more than 500 candidates (the truncation of binPhy.py:209-212; at 8
  rotations the default grid yields about 150-250 candidates, so it never truncates);
* kind 2: the no-candidate fallback rows of binPhy.py:213-224 (``select_candidates(cfg, None, ...)``: every H is the
  bin height, V from the naive mask) around a BlockOut heightmap;
* kind 3: a BlockOut observation with exactly one valid row (the mask of all other rows cleared);
* kind 4: an all-zero (idle) observation.

Before each forward ``np.random.seed(POINT_SEED)`` fixes the point indices the reference draws
(``model.py:331``); the same indices are drawn here and stored, so the shape feature can be recomputed without the
reference.  Recorded in both ``train()`` and ``eval()`` mode: the unmasked ``sum_q_map``, the masked action and the
full softmax of 4 observations.

To keep the fixture small, the network's values are chosen so that they store compactly, and are set into the
reference network BEFORE it runs (so the recorded outputs are the reference's for exactly these weights):

* every weight, bias and ``*_mu`` is rounded to ``q * 2**e`` with ``q`` an int8 per element and ``e`` one exponent per
  tensor (stored as ``q:<key>`` int8 and ``e:<key>``);
* the noise is drawn as ``NoisyLinear.reset_noise`` draws it (``model.py:214-222``) and stored by its factors:
  ``bias_epsilon`` and ``eps_in:<layer>``; ``weight_epsilon`` is their float32 outer product, bit for bit (checked
  here);
* ``*_sigma`` keep the reference's constant initialisation (``sd:<key>`` float32);
* the point clouds are multiples of 2**-10 in [0, 0.1] (``shape_array_q`` uint8).

``tests/test_actor.decode_fixture`` turns these back into the 42 ``state_dict`` arrays and ``shape_array``.
``dqn_act.npz`` as committed was written by this script with numpy 2.3.5 and
torch 2.11.
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from oracle.oracle_env import OracleConfig, OracleVecEnv, lowest_valid_action, select_candidates  # noqa: E402
from irbpp_b200 import shapes  # noqa: E402

SEL, ATOMS, POINTS = 500, 31, 1024
NET_SEED, POINT_SEED = 7, 11
SUPPORT = (-10.0, 10.0)
SOFTMAX_ROWS = (0, 5, 32, 36)            # two BlockOut bins, a fallback bin, a single-row bin
NOISY = ("fc_h_v", "fc_z_v", "fc_h_a", "fc_z_a")


def quantize(t):
    """t rounded to q * 2**e, q int8 (|q| <= 127), e the smallest exponent that keeps every |q| in range."""
    m = float(np.abs(t).max())
    e = int(np.ceil(np.log2(m / 127.0))) if m > 0 else 0
    q = np.clip(np.round(t / 2.0 ** e), -127, 127).astype(np.int8)
    return q, e


def load_model():
    ref_loader.load_reference()          # registers the stand-ins and the reference's tools module
    spec = importlib.util.spec_from_file_location("irbpp_ref_model", os.path.join(ref_loader.REFERENCE_ROOT, "model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def episode_obs(lib, R, n_envs, steps, seed, pick):
    cfg = OracleConfig(ZRotNum=R)
    env = OracleVecEnv(cfg, lib, shapes.make_sequences(n_envs, 60, lib.num_shapes, seed=seed))
    o = env.reset()
    out = []
    for t in range(steps):
        o, _, _, _ = env.step([lowest_valid_action(row, SEL) for row in o])
        out.extend(row for row in o if pick(t, row))
    return cfg, env, out


def n_valid(row):
    return int((row[:SEL * 5].reshape(SEL, 5)[:, 4] == 1).sum())


def main():
    import torch
    model = load_model()
    rng = np.random.default_rng(3)
    blk = shapes.make_blockout_library(8, seed=1)
    irr = shapes.make_irregular_library(8, seed=9, num_rotations=24)
    _, _, bobs = episode_obs(blk, 4, 6, 8, 1, lambda t, row: t in (2, 3, 5, 6))
    _, _, iobs = episode_obs(irr, 24, 12, 6, 2, lambda t, row: True)
    iobs = [r for r in iobs if np.any(r[(SEL - 1) * 5:SEL * 5] != 0)]   # the last row is filled: truncated
    obs, kinds = [], []
    for r in bobs[:20]:
        obs.append(r); kinds.append(0)
    for r in iobs[:12]:
        obs.append(r); kinds.append(1)
    cfg = OracleConfig(ZRotNum=4)
    for i in range(4):                                           # fallback rows around live heightmaps
        row = np.array(bobs[i + 6], copy=True)
        posz = rng.random((4, cfg.rangeX_A, cfg.rangeY_A))
        naive = (rng.random((4, cfg.rangeX_A, cfg.rangeY_A)) < 0.3).astype(np.float64)
        row[:SEL * 5] = select_candidates(cfg, None, posz, naive).reshape(-1)
        obs.append(row); kinds.append(2)
    for i in range(4):                                           # exactly one valid row
        row = np.array(bobs[i + 1], copy=True)
        cand = row[:SEL * 5].reshape(SEL, 5)
        keep = int(np.nonzero(cand[:, 4] == 1)[0][-1])
        cand[:, 4] = 0
        cand[keep, 4] = 1
        obs.append(row); kinds.append(3)
    for i in range(4):                                           # idle bins
        obs.append(np.zeros_like(bobs[0])); kinds.append(4)
    print("blockout", len(bobs), "irregular truncated", len(iobs))
    obs = np.stack(obs).astype(np.float32)
    kinds = np.array(kinds, np.int32)
    assert obs.shape == (44, SEL * 5 + 9 + 1024), obs.shape
    assert all(n_valid(r) == 1 for r in obs[kinds == 3])

    torch.manual_seed(NET_SEED)
    np.random.seed(NET_SEED)
    shape_q = rng.integers(0, 103, (8, 2048, 3)).astype(np.uint8)
    shape_array = (shape_q.astype(np.float32) * np.float32(2.0 ** -10))
    args = types.SimpleNamespace(selectedAction=SEL, level="location", heightMap=True, ZRotNum=4,
                                 bin_dimension=[0.32, 0.32, 0.30], resolutionH=0.01, bufferSize=1, atoms=ATOMS,
                                 hidden_size=128, noisy_std=0.5, samplePointsNum=POINTS, device=torch.device("cpu"))
    net = model.DQNBPP(args, SEL, torch.tensor(shape_array))
    out = {}
    with torch.no_grad():
        for name, mod in net.named_children():           # the compact noise: NoisyLinear.reset_noise's draw
            if name in NOISY:
                f = lambda n: (lambda x: x.sign().mul_(x.abs().sqrt_()))(torch.randn(n))
                e_in, e_out = f(mod.in_features), f(mod.out_features)
                mod.weight_epsilon.copy_(e_out.ger(e_in))
                mod.bias_epsilon.copy_(e_out)
                assert np.array_equal(np.outer(e_out.numpy(), e_in.numpy()), mod.weight_epsilon.numpy())
                out["eps_in:" + name] = e_in.numpy()
        for k, v in net.state_dict().items():             # the compact weights
            if k.endswith("weight_epsilon"):
                continue
            if "sigma" in k or k.endswith("bias_epsilon"):
                out["sd:" + k] = v.numpy()
                continue
            q, e = quantize(v.numpy())
            v.copy_(torch.tensor(q.astype(np.float32) * np.float32(2.0 ** e)))
            out["q:" + k], out["e:" + k] = q, np.int32(e)
    support = torch.linspace(SUPPORT[0], SUPPORT[1], ATOMS)
    state = torch.tensor(obs)
    mask = state[:, :SEL * 5].reshape(-1, SEL, 5)[:, :, 4]
    out.update({"obs": obs, "kinds": kinds, "shape_array_q": shape_q, "support": support.numpy(),
                "softmax_rows": np.array(SOFTMAX_ROWS, np.int32)})
    np.random.seed(POINT_SEED)
    out["point_indices"] = np.random.randint(2048, size=POINTS).astype(np.int64)
    assert len([k for k in out if k.startswith(("sd:", "q:"))]) + len(NOISY) == 42
    for mode in ("train", "eval"):
        getattr(net, mode)()
        with torch.no_grad():
            np.random.seed(POINT_SEED)
            q = net(state)                                       # model.py:386-404
            sum_q = (q * support).sum(2)                         # agent.py:54-55
            masked = sum_q.clone()
            masked[(1 - mask).bool()] = -float("inf")            # agent.py:56-57
        out[mode + "_sum_q"] = sum_q.numpy()
        out[mode + "_action"] = masked.argmax(1).numpy()
        out[mode + "_softmax"] = q[list(SOFTMAX_ROWS)].numpy()
    path = os.path.join(HERE, "dqn_act.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes; valid rows per kind:",
          {k: sorted({n_valid(r) for r in obs[kinds == k]}) for k in range(5)})


if __name__ == "__main__":
    main()
