"""The 32 x 32 action-grid fixtures of the unmodified reference (tests/golden/fine_*.npz, made by
tests/golden/make_golden_fine.py at resolutionA = resolutionH = 0.01) reproduced by the oracle (oracle/oracle_env.py,
cv2-free port) and by the kernels' Grid<1> instantiations on host threads (tests/host_harness/cuda_emu.h)."""
import ctypes

import numpy as np
import pytest

from conftest import lib_from_fixture, load_golden
from oracle.oracle_env import (HEURISTICS, OracleConfig, OracleVecEnv, convex_hull_actions, heuristic_action_port,
                               scan_vectorized)
from test_fine_grid import FineEmuEnv
from test_kernels_emulated import build_emulated, _P

pytestmark = pytest.mark.timeout(900)

RES_A = 0.01
A = 32
EPISODES = ["fine_episode_cube", "fine_episode_blockout", "fine_episode_buffered"]


def _cfg(d):
    kw = {}
    if "selectedAction" in d:
        kw = dict(selectedAction=int(d["selectedAction"]), bufferSize=int(d["bufferSize"]))
    return OracleConfig(resolutionAct=RES_A, ZRotNum=int(d["R"]), **kw)


def _check_step(t, obs, rew, done, counter, ratio, d):
    assert np.array_equal(obs, d["obs"][t + 1].astype(np.float32)), t
    assert np.array_equal(rew, d["reward"][t].astype(np.float32)) and np.array_equal(done, d["done"][t]), t
    for i in np.nonzero(d["done"][t])[0]:
        assert counter[i] == d["counter"][t][i] and ratio[i] == d["ratio"][t][i], (t, i)


# ---- the oracle against the reference --------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["cube", "irregular"])
def test_oracle_fine_scan_matches_reference(tag):
    d = load_golden("fine_scan_" + tag)
    lib = lib_from_fixture(d)
    cfg = _cfg(d)
    for k in range(len(d["item_ids"])):
        item = int(d["item_ids"][k])
        pz, pv, mk = scan_vectorized(cfg, d["heightmaps"][k], lib.extents[item], lib.tables[item])
        assert np.array_equal(pz, d["posZmap"][k]) and np.array_equal(pv, d["posZValid"][k]) and np.array_equal(mk, d["naiveMask"][k]), k


def test_oracle_fine_hulls_match_reference():
    d = load_golden("fine_hulls")
    off = 0
    assert (d["counts"] == 0).any()                        # the None fallback is among the cases
    for k in range(len(d["counts"])):
        c = int(d["counts"][k])
        got = convex_hull_actions(d["posZValid"][k][None], d["mask"][k][None], 0.01, "port")
        if c == 0:
            assert got is None, k
        else:
            assert np.array_equal(got, d["rows"][off:off + c]), k
        off += c


@pytest.mark.parametrize("name", EPISODES)
def test_oracle_fine_episodes_match_reference(name):
    d = load_golden(name)
    lib = lib_from_fixture(d)
    k = int(d["bufferSize"])
    vec = OracleVecEnv(_cfg(d), lib, d["sequences"])
    assert np.array_equal(vec.reset(), d["obs"][0])
    for t in range(len(d["actions"])):
        if k > 1:
            assert np.array_equal(np.stack(vec.get_action_candidates(d["order"][t])), d["loc_obs"][t]), t
        obs, rew, done, infos = vec.step(d["actions"][t])
        counter = [inf.get("counter", -1) for inf in infos]
        ratio = [inf.get("ratio", -1.0) for inf in infos]
        assert np.array_equal(obs, d["obs"][t + 1]), t
        assert np.array_equal(rew, d["reward"][t]) and np.array_equal(done, d["done"][t]), t
        assert counter == list(d["counter"][t]) and ratio == list(d["ratio"][t]), t
    if name == "fine_episode_blockout":                    # selectedAction 40: the truncation path ran
        assert (d["loc_obs"] if k > 1 else d["obs"])[:, :, 39 * 5 + 4].any()


def test_oracle_fine_heuristics_match_reference():
    d = load_golden("fine_heuristic")
    lib = lib_from_fixture(d)
    cfg = _cfg(d)
    vec = OracleVecEnv(cfg, lib, d["sequences"])
    assert np.array_equal(vec.reset().astype(np.float32), d["obs"][0])
    for t in range(len(d["actions"])):
        for mi, m in enumerate(HEURISTICS):
            for di in range(4):
                poses, index = vec.heuristic_actions(m, di)
                assert np.array_equal(poses, d["poses"][t, mi, di]) and np.array_equal(index, d["index"][t, mi, di]), (t, m, di)
        obs, _, done, _ = vec.step(d["actions"][t], poses=True)
        assert np.array_equal(obs.astype(np.float32), d["obs"][t + 1]) and np.array_equal(done, d["done"][t]), t


# ---- the emulated kernels against the reference --------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emulated(str(tmp_path_factory.mktemp("emu_fine_golden")))


@pytest.mark.parametrize("name,steps", [("fine_episode_cube", 24), ("fine_episode_blockout", 12), ("fine_episode_buffered", 8)])
def test_emulated_fine_episodes_match_reference(emu, name, steps):
    d = load_golden(name)
    k = int(d["bufferSize"])
    env = FineEmuEnv(emu, lib_from_fixture(d), d["sequences"], selected_action=int(d["selectedAction"]), buffer_size=k)
    assert np.array_equal(env.reset(), d["obs"][0].astype(np.float32))
    for t in range(steps):
        if k > 1:
            assert np.array_equal(env.get_action_candidates(d["order"][t]), d["loc_obs"][t].astype(np.float32)), t
        obs, r = env.step_results(d["actions"][t])
        assert not r["error"].any(), t
        _check_step(t, obs, r["reward"], r["done"].astype(bool), r["counter"], r["ratio"], d)
    env.close()


@pytest.mark.parametrize("tag", ["cube", "irregular"])
def test_emulated_fine_scan_matches_reference(emu, tag):
    d = load_golden("fine_scan_" + tag)
    lib = lib_from_fixture(d)
    n, R = len(d["item_ids"]), lib.num_rotations
    env = FineEmuEnv(emu, lib, np.zeros((n, 8), np.int32))
    assert emu.emu_irbpp_debug_set_heightmap(env.h, _P(np.ascontiguousarray(d["heightmaps"], dtype=np.float64))) == 0
    items = np.ascontiguousarray(d["item_ids"], dtype=np.int32)
    pz, pv, mk = (np.zeros((n, R, A, A)) for _ in range(3))
    cand, nh = np.zeros((n, 500, 5)), np.zeros(n, np.int32)
    assert emu.emu_irbpp_debug_scan(env.h, _P(items), _P(pz), _P(pv), _P(mk), _P(cand), _P(nh)) == 0
    assert np.array_equal(pz, d["posZmap"]) and np.array_equal(pv, d["posZValid"]) and np.array_equal(mk, d["naiveMask"])
    env.close()


def test_emulated_fine_hulls_match_reference(emu):
    """getConvexHullActions on 32 x 32 maps through irbpp_debug_hulls; where the reference returned None the table is
    the fallback and the hull count 0."""
    from irbpp_b200 import shapes
    d = load_golden("fine_hulls")
    n = len(d["counts"])
    env = FineEmuEnv(emu, shapes.make_cube_library(seed=1, num_rotations=1, num_shapes=4, resolutionAct=RES_A),
                     np.zeros((n, 8), np.int32), selected_action=1024)
    pv = np.ascontiguousarray(d["posZValid"][:, None], dtype=np.float64)
    mk = np.ascontiguousarray(d["mask"][:, None], dtype=np.float64)
    cand, nh = np.zeros((n, 1024, 5)), np.zeros(n, np.int32)
    assert emu.emu_irbpp_debug_hulls(env.h, _P(pv), _P(mk), _P(cand), _P(nh)) == 0
    off = 0
    for k in range(n):
        c = int(d["counts"][k])
        assert nh[k] == c, k
        if c:
            assert np.array_equal(cand[k, :c], d["rows"][off:off + c]), k
        off += c
    env.close()


def test_emulated_fine_heuristics_match_reference(emu):
    d = load_golden("fine_heuristic")
    env = FineEmuEnv(emu, lib_from_fixture(d), d["sequences"])
    n = env.n
    assert np.array_equal(env.reset(), d["obs"][0])
    for t in range(len(d["actions"])):
        for mi in range(4):
            for di in range(4):
                poses, index = np.zeros((n, 3), np.int32), np.zeros(n, np.int64)
                assert emu.emu_irbpp_heuristic_actions(env.h, mi, di, _P(poses), _P(index), 0, None) == 0
                assert np.array_equal(poses, d["poses"][t, mi, di]) and np.array_equal(index, d["index"][t, mi, di]), (t, mi, di)
        acts = np.ascontiguousarray(d["actions"][t], dtype=np.int64)
        obs = np.zeros((n, env.obs_len), np.float32)
        assert emu.emu_irbpp_step_poses_async(env.h, _P(acts), 0, _P(obs), None) == 0
        assert emu.emu_irbpp_step_wait(env.h, None) == 0
        assert np.array_equal(obs, d["obs"][t + 1]), t
    env.close()
