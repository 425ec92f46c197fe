"""Grouped draws and trajectory replay on the H100 (``pytest -m gpu``): the grouped stream against its Python mirror
at 4096 bins, batched ``evaluate`` against one oracle episode per trajectory and against the serial
``SingleGpuEnv`` loop of ``tools.test``, and the flagged end of a trajectory."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GROUPS = [[0], [1, 2, 3], [4, 5, 6, 7, 8], [9, 10, 11, 12, 13, 14, 15], [16, 17, 18, 19, 20, 21, 22, 23]]


def first_valid_torch(obs, sel=500):
    """Deterministic policy on the device: the first candidate row with V == 1 (row 0 if there is none)."""
    import torch
    valid = obs[:, :sel * 5].reshape(obs.shape[0], sel, 5)[:, :, 4] == 1
    return torch.argmax(valid.to(torch.int32), dim=1)


def first_valid(row, sel=500):
    v = np.nonzero(np.asarray(row[:sel * 5]).reshape(sel, 5)[:, 4] == 1)[0]
    return int(v[0]) if len(v) else 0


def test_grouped_stream_equals_mirror_at_4096_bins():
    """Every draw of 4096 bins over 101 draws (reset + 100 steps, one draw per step at k = 1) equals
    shapes.item_group_ids; group and within-group frequencies pass a chi-square test (p > 1e-3)."""
    import torch
    from scipy.stats import chisquare
    from irbpp_b200 import shapes
    from irbpp_b200.vec_env import GpuVecEnv
    lib = shapes.make_blockout_library(24, seed=31)
    n, steps, seed = 4096, 100, 1234567
    env = GpuVecEnv(lib, None, num_envs=n, item_groups=GROUPS, item_seed=seed)
    want = shapes.item_group_ids(seed, n, steps + 1, GROUPS)
    got = np.zeros_like(want)
    obs = env.reset()
    got[:, 0] = obs[:, 2500].cpu().numpy()
    for t in range(steps):
        obs, _, _, _ = env.step(first_valid_torch(obs))
        got[:, t + 1] = obs[:, 2500].cpu().numpy()
    env.close()
    assert np.array_equal(got, want)
    gid = np.zeros(lib.num_shapes, np.int64)
    for g, ids in enumerate(GROUPS):
        gid[ids] = g
    counts = np.bincount(gid[got.reshape(-1)], minlength=len(GROUPS))
    assert chisquare(counts).pvalue > 1e-3
    for ids in GROUPS[1:]:
        c = np.bincount(got.reshape(-1), minlength=lib.num_shapes)[ids]
        assert chisquare(c).pvalue > 1e-3, ids
    torch.cuda.synchronize()


def test_grouped_episodes_match_oracle_stream():
    """item_groups: the oracle is given the mirrored stream as an explicit, long-enough sequence."""
    from irbpp_b200 import shapes
    from irbpp_b200.vec_env import GpuVecEnv
    from oracle.oracle_env import OracleConfig, OracleVecEnv
    lib = shapes.make_blockout_library(24, seed=31)
    n, steps, seed = 40, 50, 20261015
    stream = shapes.item_group_ids(seed, n, 4 * steps + 8, GROUPS)
    ora = OracleVecEnv(OracleConfig(ZRotNum=4), lib, stream)
    env = GpuVecEnv(lib, None, num_envs=n, item_groups=GROUPS, item_seed=seed)
    o_obs = ora.reset()
    assert np.array_equal(env.reset().cpu().numpy(), o_obs.astype(np.float32))
    rng = np.random.default_rng(6)
    for t in range(steps):
        acts = np.zeros(n, dtype=np.int64)
        for i in range(n):
            valid = np.nonzero(o_obs[i][:2500].reshape(500, 5)[:, 4] == 1)[0]
            acts[i] = int(rng.choice(valid)) if len(valid) else 0
        o_obs, _, o_done, _ = ora.step(acts)
        g_obs, _, g_done, _ = env.step(acts)
        assert np.array_equal(g_obs.cpu().numpy(), o_obs.astype(np.float32)), t
        assert np.array_equal(g_done, o_done)
    assert np.array_equal(env.debug_state()["cursor"], [e.cursor for e in ora.envs])
    env.close()


def _trajectories(lib, count, seed):
    rng = np.random.default_rng(seed)
    return [[int(v) for v in rng.integers(0, lib.num_shapes, size=int(rng.integers(30, 40)))] for _ in range(count)]


def _oracle_episode(lib, traj, k):
    """One tools.test / tools.test_hierachical episode of the oracle: (reward sum, length, ratio, counter)."""
    from oracle.oracle_env import OracleConfig, OracleEnv
    o = OracleEnv(OracleConfig(ZRotNum=lib.num_rotations, bufferSize=k), lib, traj)
    obs = o.reset()
    rsum, n = 0.0, 0
    while True:
        if k > 1:
            obs = o.get_action_candidates(int(np.argmax(obs[:k])))
        obs, r, d, info = o.step(first_valid(obs))
        rsum += r
        n += 1
        if d:
            return rsum, n, info["ratio"], info["counter"]


@pytest.mark.parametrize("k", [1, 3])
def test_evaluate_matches_oracle_and_serial_env(k):
    """evaluate over trajectories 1..300 on 64 bins equals one oracle episode per trajectory (every trajectory) and
    the serial SingleGpuEnv loop of tools.test from first_trajectory=1 (the first 12)."""
    import torch
    from irbpp_b200 import shapes
    from irbpp_b200.evaluation import evaluate
    from irbpp_b200.single_env import SingleGpuEnv
    lib = shapes.make_blockout_library(10, seed=8, edge=0.08)
    trajs = _trajectories(lib, 301, seed=k)
    order = (lambda obs: torch.argmax(obs[:, :k], dim=1)) if k > 1 else None
    res = evaluate(lib, trajs, first_valid_torch, 64, first=1, count=300, order_policy=order, buffer_size=k)
    assert list(res["trajectory"]) == list(range(1, 301))
    for i, t in enumerate(range(1, 301)):
        rsum, n, ratio, counter = _oracle_episode(lib, trajs[t], k)
        assert (res["reward_sum"][i], res["length"][i], res["ratio"][i], res["counter"][i]) == (rsum, n, ratio, counter), t
    assert res["summary"]["avg_length"] == np.mean(res["length"])
    env = SingleGpuEnv(lib, trajectories=trajs, first_trajectory=1, buffer_size=k)
    for j in range(12):
        state, rsum, n = env.reset(), 0.0, 0
        assert env.item_creator.traj_index == 1 + j
        while True:
            if k > 1:
                state = env.get_action_candidates(int(np.argmax(state[:k])))
            state, r, done, _ = env.step(first_valid(state))
            rsum += r
            n += 1
            if done:
                break
        assert (n, env.get_ratio()) == (res["length"][j], res["ratio"][j]), j
        assert abs(rsum - res["reward_sum"][j]) < 1e-4          # tools.test sums the float32 step rewards
    env.close()


def test_trajectory_end_is_flagged_error_5():
    """A trajectory shorter than what its bin places: step_wait raises IRBPP_EDEVICE naming the bin and code 5."""
    from irbpp_b200 import _lib, shapes
    from irbpp_b200.vec_env import GpuVecEnv
    lib = shapes.make_blockout_library(10, seed=8)
    trajs = [[1, 2, 3, 4, 5, 6, 7, 8]] * 5 + [[1, 2]] + [[1, 2, 3, 4, 5, 6, 7, 8]] * 2
    env = GpuVecEnv(lib, None, num_envs=8, trajectories=trajs, first_trajectory=0)
    obs = env.reset()
    obs, _, done, _ = env.step(first_valid_torch(obs))
    assert not done.any()
    with pytest.raises(_lib.IrbppError) as ei:
        env.step(first_valid_torch(obs))
    assert ei.value.code == _lib.IRBPP_EDEVICE and "env 5 reported device error code 5" in str(ei.value)
    env.close()
