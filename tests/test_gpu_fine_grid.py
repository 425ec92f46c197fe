"""The 32 x 32 action grid (resolutionA = resolutionH = 0.01) on the H100 (``pytest -m gpu``): GpuVecEnv at 4096 Cube
bins against the oracle on a sample of bins through auto-resets, BlockOut shapes with truncation, the buffered
protocol, heuristics and explicit poses, debug views, and trajectory replay with idle bins -- value-exact, as the
16 x 16 tests are."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RES_A = 0.01
A = 32


def _env(lib, seqs, **kw):
    from irbpp_b200.vec_env import GpuVecEnv
    return GpuVecEnv(lib, seqs, device=kw.pop("device", "cuda:0"), **kw)


def _cfg(lib, **kw):
    from oracle.oracle_env import OracleConfig
    return OracleConfig(resolutionAct=RES_A, ZRotNum=lib.num_rotations, **kw)


def _random_valid(rng, rows, sel):
    valid = np.nonzero(np.asarray(rows[:sel * 5]).reshape(sel, 5)[:, 4] == 1)[0]
    return int(rng.choice(valid)) if len(valid) else 0


def test_fine_cube_4096_bins_sampled_against_oracle():
    """4096 Cube bins (R = 2) under a random valid policy for 40 steps; 12 sampled bins are replayed by the oracle and
    must match observation row, reward, done and, at the end of an episode, counter and ratio -- auto-resets included."""
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleEnv
    lib = shapes.make_cube_library(seed=3, num_rotations=2, resolutionAct=RES_A)
    n, sel = 4096, 500
    seqs = shapes.make_sequences(n, 96, lib.num_shapes, seed=5)
    env = _env(lib, seqs)
    assert (env.Ax, env.Ay) == (A, A)
    sample = np.linspace(0, n - 1, 12).astype(int)
    cfg = _cfg(lib)
    oracles = {i: OracleEnv(cfg, lib, seqs[i]) for i in sample}
    obs = env.reset().cpu().numpy()
    for i, o in oracles.items():
        assert np.array_equal(obs[i], o.reset().astype(np.float32)), i
    rng = np.random.default_rng(0)
    dones = 0
    for t in range(40):
        acts = np.array([_random_valid(rng, obs[i], sel) for i in range(n)], dtype=np.int64)
        g, rew, done, infos = env.step(acts)
        obs = g.cpu().numpy()
        for i, o in oracles.items():
            w, r, d, info = o.step(int(acts[i]))
            if d:
                assert infos[i]["counter"] == info["counter"] and infos[i]["ratio"] == info["ratio"], (t, i)
                w = o.reset()
            assert np.array_equal(obs[i], w.astype(np.float32)), (t, i)
            assert np.float32(r) == rew[i, 0].item() and bool(d) == bool(done[i]), (t, i)
            dones += int(d)
    assert dones > 0
    env.close()


@pytest.mark.parametrize("k", [1, 5])
def test_fine_blockout_truncation_and_buffered(k):
    """BlockOut shapes (R = 4) with a 40-row table (every step truncates) online, and the buffered protocol (k = 5:
    get_all_possible_observation, get_action_candidates, order observations), all bins against the oracle."""
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleVecEnv
    lib = shapes.make_blockout_library(12, seed=4, resolutionAct=RES_A)
    n, sel = 64, 40
    seqs = shapes.make_sequences(n, 64, lib.num_shapes, seed=6)
    env = _env(lib, seqs, selected_action=sel, buffer_size=k)
    ora = OracleVecEnv(_cfg(lib, selectedAction=sel, bufferSize=k), lib, seqs)
    want = ora.reset()
    assert np.array_equal(env.reset().cpu().numpy(), want.astype(np.float32))
    rng = np.random.default_rng(k)
    for t in range(10):
        loc = want
        if k > 1:
            all_o = np.stack([e.get_all_possible_observation() for e in ora.envs])
            assert np.array_equal(env.get_all_possible_observation().cpu().numpy(), all_o.astype(np.float32)), t
            order = rng.integers(0, k, size=n)
            loc = np.stack(ora.get_action_candidates(order))
            assert np.array_equal(env.get_action_candidates(order, as_tensor=True).cpu().numpy(), loc.astype(np.float32)), t
        acts = np.array([_random_valid(rng, loc[i], sel) for i in range(n)], dtype=np.int64)
        want, rew, done, _ = ora.step(acts)
        g, grew, gdone, _ = env.step(acts)
        assert np.array_equal(g.cpu().numpy(), want.astype(np.float32)), t
        assert np.array_equal(grew.numpy()[:, 0], rew.astype(np.float32)) and np.array_equal(gdone, done), t
    env.close()


def test_fine_heuristics_step_poses_and_debug_views():
    """The four heuristics in four directions and step_poses ([N, 3] and flat) on irregular shapes, then the debug
    views shaped [N, R, 32, 32], against the oracle."""
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleVecEnv, convex_hull_actions, scan_vectorized
    lib = shapes.make_irregular_library(8, seed=7, num_rotations=2, resolutionAct=RES_A)
    n = 16
    seqs = shapes.make_sequences(n, 48, lib.num_shapes, seed=8)
    env = _env(lib, seqs)
    ora = OracleVecEnv(_cfg(lib), lib, seqs)
    want = ora.reset()
    assert np.array_equal(env.reset().cpu().numpy(), want.astype(np.float32))
    for t in range(6):
        for m in env.HEURISTICS:
            for d in range(4):
                poses, index = env.get_heuristic_actions(m, d)
                wp, wi = ora.heuristic_actions(m, d)
                assert np.array_equal(poses, wp) and np.array_equal(index, wi), (t, m, d)
        poses, _ = env.get_heuristic_actions(env.HEURISTICS[t % 4])
        flat = (poses[:, 0].astype(np.int64) * A + poses[:, 1]) * A + poses[:, 2]
        want, rew, done, _ = ora.step(flat, poses=True)
        g, grew, gdone, _ = env.step_poses(poses if t % 2 else flat)
        assert np.array_equal(g.cpu().numpy(), want.astype(np.float32)), t
        assert np.array_equal(gdone, done), t
    cfg = _cfg(lib)
    rng = np.random.default_rng(2)
    hm = np.round(rng.random((n, 32, 32)) * 0.1, 3)
    env.debug_set_heightmap(hm)
    items = rng.integers(0, lib.num_shapes, size=n)
    out = env.debug_scan(items)
    assert out["posZmap"].shape == (n, 2, A, A)
    for i in range(n):
        wz, wv, wm = scan_vectorized(cfg, hm[i], lib.extents[items[i]], lib.tables[items[i]])
        assert np.array_equal(out["posZmap"][i], wz) and np.array_equal(out["naiveMask"][i], wm), i
        hull = convex_hull_actions(wv, wm, 0.01, "port")
        assert out["num_hull"][i] == (0 if hull is None else len(hull)), i
    hv = env.debug_hulls(out["posZValid"], out["naiveMask"])
    assert np.array_equal(hv["num_hull"], out["num_hull"]) and np.array_equal(hv["cand"], out["cand"])
    env.close()


def test_fine_trajectory_replay_with_idle_bins():
    """Trajectory replay on the 32 x 32 grid: 8 trajectories on 6 bins, so bins turn idle; every live bin's episode
    equals the oracle's, idle bins give zero rows and Valid False."""
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleEnv
    lib = shapes.make_cube_library(seed=9, num_rotations=2, resolutionAct=RES_A)
    rng = np.random.default_rng(4)
    trajs = [[int(v) for v in rng.integers(0, lib.num_shapes, size=300)] for _ in range(9)]
    n = 6
    env = _env(lib, None, num_envs=n, trajectories=trajs, first_trajectory=1)
    cfg = _cfg(lib)
    obs = env.reset().cpu().numpy()
    oracles = {}
    for i in range(n):
        oracles[i] = OracleEnv(cfg, lib, trajs[env.trajectory[i]])
        assert np.array_equal(obs[i], oracles[i].reset().astype(np.float32)), i
    idle_seen = False
    for t in range(80):
        acts = np.array([_random_valid(rng, obs[i], 500) for i in range(n)], dtype=np.int64)
        was_idle = env.idle.copy()
        g, rew, done, infos = env.step(acts)
        obs = g.cpu().numpy()
        for i in range(n):
            if was_idle[i]:
                assert not infos[i]["Valid"] and not np.any(obs[i]) and not done[i], (t, i)
                idle_seen = True
                continue
            w, r, d, info = oracles[i].step(int(acts[i]))
            assert bool(d) == bool(done[i]) and np.float32(r) == rew[i, 0].item(), (t, i)
            if d:
                assert infos[i]["counter"] == info["counter"] and infos[i]["ratio"] == info["ratio"], (t, i)
                if env.idle[i]:
                    assert not np.any(obs[i]), (t, i)
                    continue
                oracles[i] = OracleEnv(cfg, lib, trajs[env.trajectory[i]])
                w = oracles[i].reset()
            assert np.array_equal(obs[i], w.astype(np.float32)), (t, i)
    assert idle_seen
    env.close()


@pytest.mark.parametrize("name", ["fine_episode_cube", "fine_episode_blockout", "fine_episode_buffered"])
def test_fine_reference_episodes(name):
    """The reference's 32 x 32 episodes (tests/golden/make_golden_fine.py) through GpuVecEnv, every step."""
    from conftest import lib_from_fixture, load_golden
    d = load_golden(name)
    k = int(d["bufferSize"])
    env = _env(lib_from_fixture(d), d["sequences"], selected_action=int(d["selectedAction"]), buffer_size=k)
    assert np.array_equal(env.reset().cpu().numpy(), d["obs"][0].astype(np.float32))
    for t in range(len(d["actions"])):
        if k > 1:
            got = env.get_action_candidates(d["order"][t], as_tensor=True).cpu().numpy()
            assert np.array_equal(got, d["loc_obs"][t].astype(np.float32)), t
        g, rew, done, infos = env.step(np.ascontiguousarray(d["actions"][t], dtype=np.int64))
        assert np.array_equal(g.cpu().numpy(), d["obs"][t + 1].astype(np.float32)), t
        assert np.array_equal(rew.numpy()[:, 0], d["reward"][t].astype(np.float32)) and np.array_equal(done, d["done"][t]), t
        for i in np.nonzero(d["done"][t])[0]:
            assert infos[i]["counter"] == d["counter"][t][i] and infos[i]["ratio"] == d["ratio"][t][i], (t, i)
    env.close()


def test_fine_reference_scan_hulls_and_heuristics():
    """The reference's 32 x 32 scan cases, getConvexHullActions maps (None cases included) and heuristic episode
    through GpuVecEnv's debug views, get_heuristic_actions and step_poses."""
    from irbpp_b200 import shapes
    from conftest import lib_from_fixture, load_golden
    for tag in ("cube", "irregular"):
        d = load_golden("fine_scan_" + tag)
        n = len(d["item_ids"])
        env = _env(lib_from_fixture(d), np.zeros((n, 8), np.int32))
        env.debug_set_heightmap(d["heightmaps"])
        out = env.debug_scan(d["item_ids"])
        assert np.array_equal(out["posZmap"], d["posZmap"]) and np.array_equal(out["posZValid"], d["posZValid"])
        assert np.array_equal(out["naiveMask"], d["naiveMask"]), tag
        env.close()
    d = load_golden("fine_hulls")
    n = len(d["counts"])
    env = _env(shapes.make_cube_library(seed=1, num_rotations=1, num_shapes=4, resolutionAct=RES_A), np.zeros((n, 8), np.int32),
               selected_action=1024)
    out = env.debug_hulls(d["posZValid"][:, None], d["mask"][:, None])
    off = 0
    for k in range(n):
        c = int(d["counts"][k])
        assert out["num_hull"][k] == c, k
        if c:
            assert np.array_equal(out["cand"][k, :c], d["rows"][off:off + c]), k
        off += c
    env.close()
    d = load_golden("fine_heuristic")
    env = _env(lib_from_fixture(d), d["sequences"])
    assert np.array_equal(env.reset().cpu().numpy(), d["obs"][0])
    for t in range(len(d["actions"])):
        for mi, m in enumerate(env.HEURISTICS):
            for di in range(4):
                poses, index = env.get_heuristic_actions(m, di)
                assert np.array_equal(poses, d["poses"][t, mi, di]) and np.array_equal(index, d["index"][t, mi, di]), (t, m, di)
        g, _, done, _ = env.step_poses(d["actions"][t])
        assert np.array_equal(g.cpu().numpy(), d["obs"][t + 1]) and np.array_equal(done, d["done"][t]), t
    env.close()
