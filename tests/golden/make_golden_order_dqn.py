"""Generate ``dqn_order_act.npz`` from the UNMODIFIED reference order network (``model.py`` ``DQNBPP`` with
``args.level = 'order'`` and ``bufferSize`` k) and ``Agent.act`` (``agent.py:51-58``; the reference passes no mask at
this level).

Run in the build container (needs the reference tree and torch):

    python tests/golden/make_golden_order_dqn.py

``model.py`` is executed from where it lies, after ``oracle/ref_loader.py`` has installed its import stand-ins.  One
seeded ``DQNBPP(args, 10, shapeArray)`` (atoms 31, hidden 128, noisy_std 0.5) is built; a second one with
``bufferSize = 3`` loads its state dict (the graph size is fixed at construction, the weights are not).  Both run on
the CPU in float32 over order observations ``[k item ids | heightmap]`` of ``OracleVecEnv(bufferSize=k)`` mid-episode
(order action: a seeded random slot; location action: the lowest valid candidate), plus two idle all-zero rows each.

Point clouds: the order level keeps a 10 000-point subsample of every cloud (``model.py:242-244, 301-306``) and each
forward draws 1024 of those points (``:367-368``).  Here ``np.random.seed(SUBSAMPLE_SEED)`` precedes a call of the
reference's own ``updateShapeArray`` and ``np.random.seed(POINT_SEED)`` every forward; the same draws are repeated
here, and their composition (``subsample[draw]``, indices into the full clouds) is stored as ``point_indices`` with
only the points it selects (``clouds_q``, ``[S, 1024, 3]`` uint8 in steps of 2**-10): the shape feature needs nothing
else.  Recorded in both ``train()`` and ``eval()`` mode for k = 3 and k = 10: ``sum_q_map``, the action and the full
softmax of 3 observations.

Weights, noise and clouds are stored compactly exactly as ``make_golden_dqn.py`` stores them (int8 times a power of
two per tensor, set into the network BEFORE it runs; the noise by its factors; ``*_sigma`` as float32); all 55
``state_dict`` keys of the order-level network are recorded, ``init_candidate_embed`` and ``project_layer`` (unused at
this level) as zeros.  ``tests/test_order_actor.decode_fixture`` turns them
back into arrays.  ``dqn_order_act.npz`` as committed was written by this script with numpy 2.3.5 and torch 2.11.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_dqn import NOISY, load_model, quantize  # noqa: E402
from oracle.oracle_env import OracleConfig, OracleVecEnv, lowest_valid_action  # noqa: E402
from irbpp_b200 import shapes  # noqa: E402

KS = (3, 10)
ATOMS, POINTS, ARRAY_POINTS = 31, 1024, 10000
NET_SEED, SUBSAMPLE_SEED, POINT_SEED = 7, 13, 11
SUPPORT = (-10.0, 10.0)
SOFTMAX_ROWS = (0, 5, 9)
UNUSED = ("init_candidate_embed.", "project_layer.")      # in the state dict, unused at the order level: stored as zeros


def order_obs(lib, k, n_envs, steps, seed):
    """Order observations of n_envs bins over ``steps`` hierarchical steps (rows of steps 2, 4, ...)."""
    cfg = OracleConfig(ZRotNum=4, bufferSize=k)
    env = OracleVecEnv(cfg, lib, shapes.make_sequences(n_envs, 80, lib.num_shapes, seed=seed))
    rng = np.random.default_rng(seed)
    o = env.reset()
    out = []
    for t in range(steps):
        if t >= 2 and t % 2 == 0:
            out.extend(np.array(row, np.float32) for row in o)
        order = rng.integers(0, k, n_envs)
        loc = env.get_action_candidates(order)
        o, _, _, _ = env.step([lowest_valid_action(row, cfg.selectedAction) for row in loc])
    return out


def main():
    import torch
    model = load_model()
    lib = shapes.make_blockout_library(8, seed=1)
    S = lib.num_shapes
    rng = np.random.default_rng(5)
    torch.manual_seed(NET_SEED)
    np.random.seed(NET_SEED)
    shape_q = rng.integers(0, 103, (S, ARRAY_POINTS, 3)).astype(np.uint8)
    shape_array = shape_q.astype(np.float32) * np.float32(2.0 ** -10)

    def args(k):
        return types.SimpleNamespace(selectedAction=500, level="order", heightMap=True, ZRotNum=4,
                                     bin_dimension=[0.32, 0.32, 0.30], resolutionH=0.01, bufferSize=k, atoms=ATOMS,
                                     hidden_size=128, noisy_std=0.5, samplePointsNum=POINTS, device=torch.device("cpu"))

    net = model.DQNBPP(args(KS[1]), KS[1], torch.tensor(shape_array))
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
            if k.startswith(UNUSED):
                v.zero_()
            q, e = quantize(v.numpy())
            v.copy_(torch.tensor(q.astype(np.float32) * np.float32(2.0 ** e)))
            out["q:" + k], out["e:" + k] = q, np.int32(e)
    assert len([k for k in out if k.startswith(("sd:", "q:"))]) + len(NOISY) == len(net.state_dict()) == 55
    # the subsample (model.py:301-306), by the reference's own method
    np.random.seed(SUBSAMPLE_SEED)
    net.updateShapeArray()
    np.random.seed(SUBSAMPLE_SEED)
    sub = np.random.randint(ARRAY_POINTS, size=ARRAY_POINTS)
    assert np.array_equal(net.shapeArray.numpy(), shape_array[:, sub])
    np.random.seed(POINT_SEED)
    composed = sub[np.random.randint(ARRAY_POINTS, size=POINTS)]
    support = torch.linspace(SUPPORT[0], SUPPORT[1], ATOMS)
    out.update({"point_indices": composed.astype(np.int64), "clouds_q": shape_q[:, composed],
                "support": support.numpy(), "softmax_rows": np.array(SOFTMAX_ROWS, np.int32)})
    for k in KS:
        if k == KS[1]:
            netk = net
        else:
            netk = model.DQNBPP(args(k), k, torch.tensor(shape_array))
            netk.load_state_dict(net.state_dict())
            netk.shapeArray = net.shapeArray.clone()
        rows = order_obs(lib, k, 4, 8, seed=k)
        obs = np.stack(rows + [np.zeros_like(rows[0])] * 2).astype(np.float32)
        assert obs.shape[1] == k + 1024
        state = torch.tensor(obs)
        out["obs%d" % k] = obs
        for mode in ("train", "eval"):
            getattr(netk, mode)()
            with torch.no_grad():
                np.random.seed(POINT_SEED)
                q = netk(state)                                   # model.py:386-404
                sum_q = (q * support).sum(2)                      # agent.py:54-55
            out["%s_sum_q%d" % (mode, k)] = sum_q.numpy()
            out["%s_action%d" % (mode, k)] = sum_q.argmax(1).numpy()
            out["%s_softmax%d" % (mode, k)] = q[list(SOFTMAX_ROWS)].numpy()
        print("k %d: %d observations" % (k, obs.shape[0]))
    path = os.path.join(HERE, "dqn_order_act.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
