"""GPU parity tests (run on an H100: ``pytest -m gpu``).  Every check goes through the C ABI
(ctypes -> libirbpp.so -> irbpp_scan_kernel / irbpp_candidates_kernel) and compares with (a) the committed outputs of the
UNMODIFIED reference (tests/golden) and (b) the oracle on the same seeded inputs.  Bar: value-exact
(``np.array_equal``; -0.0 == +0.0, SURVEY.md 8c) for every float64 view and for the float32
observations against the float32 cast of the reference's float64 observations (envs.py:151,163)."""
import numpy as np
import pytest

from conftest import lib_from_fixture, load_golden

pytestmark = pytest.mark.gpu


def _env(lib, seqs, **kw):
    from irbpp_b200.vec_env import GpuVecEnv
    return GpuVecEnv(lib, seqs, device="cuda:0", **kw)


def _dummy_seqs(n, lib, length=8):
    return np.zeros((n, length), dtype=np.int32)


@pytest.mark.parametrize("tag", ["blockout", "irregular", "cube"])
def test_scan_matches_reference_golden(tag):
    d = load_golden("scan_" + tag)
    lib = lib_from_fixture(d)
    n = len(d["item_ids"])
    env = _env(lib, _dummy_seqs(n, lib))
    env.debug_set_heightmap(d["heightmaps"])
    out = env.debug_scan(d["item_ids"])
    assert np.array_equal(out["posZmap"], d["posZmap"])
    assert np.array_equal(out["posZValid"], d["posZValid"])
    assert np.array_equal(out["naiveMask"], d["naiveMask"])
    # and the heightmaps round-trip through the device layout untouched
    assert np.array_equal(env.debug_state()["heightmap"], d["heightmaps"])
    env.close()


def test_hull_actions_match_reference_golden():
    from irbpp_b200 import shapes
    d = load_golden("hulls")
    n = len(d["counts"])
    lib = shapes.make_cube_library(seed=1, num_rotations=1, num_shapes=4)
    env = _env(lib, _dummy_seqs(n, lib), selected_action=256)
    out = env.debug_hulls(d["posZValid"][:, None], d["mask"][:, None])
    off = 0
    for k in range(n):
        c = int(d["counts"][k])
        assert out["num_hull"][k] == c, k
        if c:
            assert np.array_equal(out["cand"][k, :c], d["rows"][off:off + c]), k
            assert not out["cand"][k, c:].any()
        off += c
    env.close()


def test_hull_actions_legacy_switch_matches_oracle():
    """approx_legacy=1 selects the point-to-line rule (unpinned against the reference's cv2 4.4.0.46;
    checked against the oracle's restatement of that rule)."""
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleConfig
    from oracle import contours_port
    d = load_golden("hulls")
    n = len(d["counts"])
    lib = shapes.make_cube_library(seed=1, num_rotations=1, num_shapes=4)
    env = _env(lib, _dummy_seqs(n, lib), selected_action=256, approx_legacy=True)
    out = env.debug_hulls(d["posZValid"][:, None], d["mask"][:, None])
    for k in range(n):
        hulls, V = contours_port.convex_hulls_port(d["posZValid"][k], d["mask"][k], 0.01, legacy_line_distance=True)
        assert out["num_hull"][k] == len(hulls), k
        for i in range(len(hulls)):
            assert out["cand"][k, i, 1] == hulls[i][1] and out["cand"][k, i, 2] == hulls[i][0]
    env.close()


def _check_step(out, d, t, tag):
    obs, rew, done, infos = out
    want_obs = d["obs"][t + 1].astype(np.float32)
    got = obs.cpu().numpy()
    assert np.array_equal(got, want_obs), (tag, t, np.argwhere(got != want_obs)[:5])
    assert np.array_equal(rew.numpy()[:, 0], d["reward"][t].astype(np.float32)), (tag, t)
    assert np.array_equal(done, d["done"][t]), (tag, t)
    for i in range(len(done)):
        info = infos[i]
        assert info["Valid"] is True
        if done[i]:
            assert info["counter"] == d["counter"][t][i]
            assert info["ratio"] == d["ratio"][t][i]
            assert info["episode"]["r"] == d["ep_r"][t][i]
            assert info["episode"]["l"] == d["ep_l"][t][i]
        else:
            assert "episode" not in info


@pytest.mark.parametrize("name", ["episode_blockout", "episode_irregular", "episode_cube", "episode_truncate",
                                  "episode_rot24"])
def test_episode_matches_reference_golden(name):
    d = load_golden(name)
    lib = lib_from_fixture(d)
    env = _env(lib, d["sequences"], selected_action=int(d["selectedAction"]))
    obs = env.reset()
    assert obs.dtype.is_floating_point and tuple(obs.shape) == d["obs"][0].shape and obs.is_cuda
    assert np.array_equal(obs.cpu().numpy(), d["obs"][0].astype(np.float32))
    for t in range(len(d["actions"])):
        _check_step(env.step(d["actions"][t]), d, t, name)
    env.close()


def test_buffered_episode_matches_reference_golden():
    d = load_golden("episode_buffered")
    lib = lib_from_fixture(d)
    env = _env(lib, d["sequences"], buffer_size=int(d["bufferSize"]))
    obs = env.reset()
    assert np.array_equal(obs.cpu().numpy(), d["obs"][0].astype(np.float32))
    for t in range(len(d["actions"])):
        loc = env.get_action_candidates(d["order"][t])
        assert isinstance(loc, list) and loc[0].dtype == np.float64            # reference return type
        assert np.array_equal(np.stack(loc), d["loc_obs"][t].astype(np.float32).astype(np.float64)), t
        _check_step(env.step(d["actions"][t]), d, t, "buffered")
    env.close()


def _random_valid_actions(rng, loc_obs, sel):
    acts = np.zeros(len(loc_obs), dtype=np.int64)
    for i in range(len(loc_obs)):
        cand = loc_obs[i][:sel * 5].reshape(sel, 5)
        valid = np.nonzero(cand[:, 4] == 1)[0]
        acts[i] = int(rng.choice(valid)) if len(valid) else 0
    return acts


@pytest.mark.parametrize("kind,R,n_envs,steps", [("blockout", 4, 48, 60), ("irregular", 8, 32, 40), ("cube", 2, 32, 50)])
def test_random_episodes_match_oracle(kind, R, n_envs, steps):
    """Seeded random-valid policy; CUDA path vs the oracle, step by step, including auto-resets."""
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleConfig, OracleVecEnv
    lib = {"blockout": lambda: shapes.make_blockout_library(24, seed=31),
           "irregular": lambda: shapes.make_irregular_library(24, seed=32),
           "cube": lambda: shapes.make_cube_library(seed=33, num_shapes=30)}[kind]()
    seqs = shapes.make_sequences(n_envs, 40, lib.num_shapes, seed=77)
    cfg = OracleConfig(ZRotNum=R)
    ora = OracleVecEnv(cfg, lib, seqs)
    env = _env(lib, seqs)
    o_obs = ora.reset()
    g_obs = env.reset()
    assert np.array_equal(g_obs.cpu().numpy(), o_obs.astype(np.float32))
    rng = np.random.default_rng(5)
    n_done = 0
    for t in range(steps):
        acts = _random_valid_actions(rng, o_obs, 500)
        o_obs, o_rew, o_done, o_infos = ora.step(acts)
        g_obs, g_rew, g_done, g_infos = env.step(acts)
        assert np.array_equal(g_obs.cpu().numpy(), o_obs.astype(np.float32)), (kind, t)
        assert np.array_equal(g_rew.numpy()[:, 0], o_rew.astype(np.float32))
        assert np.array_equal(g_done, o_done)
        for i in np.nonzero(o_done)[0]:
            gi, oi = g_infos[int(i)], o_infos[int(i)]
            assert gi["counter"] == oi["counter"] and gi["ratio"] == oi["ratio"]
            assert gi["episode"]["r"] == oi["episode"]["r"] and gi["episode"]["l"] == oi["episode"]["l"]
        n_done += int(o_done.sum())
    st = env.debug_state()
    assert np.array_equal(st["heightmap"], np.stack([e.heightmap for e in ora.envs]))
    assert n_done > 0
    env.close()


def test_get_all_possible_observation_matches_oracle():
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleConfig, OracleVecEnv
    lib = shapes.make_blockout_library(16, seed=41)
    seqs = shapes.make_sequences(6, 32, lib.num_shapes, seed=3)
    k = 4
    cfg = OracleConfig(ZRotNum=4, bufferSize=k)
    ora = OracleVecEnv(cfg, lib, seqs)
    env = _env(lib, seqs, buffer_size=k)
    ora.reset(); env.reset()
    rng = np.random.default_rng(0)
    for t in range(12):
        want = np.stack([e.get_all_possible_observation() for e in ora.envs])
        got = env.get_all_possible_observation().cpu().numpy()
        assert np.array_equal(got, want.astype(np.float32)), t
        order = rng.integers(0, k, size=6)
        loc = np.stack(ora.get_action_candidates(order))
        gloc = env.get_action_candidates(order, as_tensor=True).cpu().numpy()
        assert np.array_equal(gloc, loc.astype(np.float32))
        acts = _random_valid_actions(rng, loc, 500)
        o = ora.step(acts); g = env.step(acts)
        assert np.array_equal(g[0].cpu().numpy(), o[0].astype(np.float32))
        assert np.array_equal(g[2], o[2])
    env.close()


def test_vec_env_contract():
    """Call-order errors and return types of the VecEnv surface (wrapper/vec_env.py:7-26,101-108;
    envs.py:149-165)."""
    import torch
    from irbpp_b200 import shapes
    from irbpp_b200.vec_env import AlreadySteppingError, NotSteppingError
    lib = shapes.make_blockout_library(8, seed=1)
    seqs = shapes.make_sequences(5, 16, lib.num_shapes, seed=1)
    env = _env(lib, seqs)
    assert env.num_envs == 5 and env.observation_space.shape == (3533,) and env.action_space.n == 500
    with pytest.raises(NotSteppingError):
        env.step_wait()
    obs = env.reset()
    assert obs.dtype == torch.float32 and obs.shape == (5, 3533) and obs.device.type == "cuda"
    env.step_async(np.zeros(5, dtype=np.int64))
    with pytest.raises(AlreadySteppingError):
        env.step_async(np.zeros(5, dtype=np.int64))
    obs, rew, done, infos = env.step_wait()
    assert rew.dtype == torch.float32 and rew.shape == (5, 1) and rew.device.type == "cpu"
    assert done.dtype == np.bool_ and done.shape == (5,)
    assert len(infos) == 5 and all("Valid" in infos[i] for i in range(5))
    # CUDA tensor actions (trainer passes action.cpu().numpy(); both must work), and [N,1] LongTensor
    obs2, _, _, _ = env.step(torch.zeros((5, 1), dtype=torch.int64, device="cuda:0"))
    assert obs2.shape == (5, 3533)
    with pytest.raises(ValueError):
        env.step(np.zeros(4, dtype=np.int64))
    from irbpp_b200._lib import IrbppError
    with pytest.raises(IrbppError):
        env.step(np.full(5, 500, dtype=np.int64))     # action outside the candidate table
    env.close()


def test_reset_specific_and_sequence_wrap():
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleConfig, OracleEnv
    lib = shapes.make_blockout_library(8, seed=2)
    seqs = shapes.make_sequences(4, 5, lib.num_shapes, seed=9)     # short: the cursor wraps
    env = _env(lib, seqs)
    obs = env.reset()
    cfg = OracleConfig(ZRotNum=4)
    oracles = [OracleEnv(cfg, lib, seqs[i]) for i in range(4)]
    want = np.stack([o.reset() for o in oracles])
    assert np.array_equal(obs.cpu().numpy(), want.astype(np.float32))
    before = obs.clone()
    env.reset_specific([1, 3], obs)
    for i in (1, 3):
        want[i] = oracles[i].reset()
    got = obs.cpu().numpy()
    assert np.array_equal(got, want.astype(np.float32))
    assert np.array_equal(got[0], before[0].cpu().numpy()) and np.array_equal(got[2], before[2].cpu().numpy())
    for t in range(12):                                             # > 5 draws per env -> wrap-around
        acts = np.array([int(np.argmax(want[i][:2500].reshape(500, 5)[:, 4] == 1)) for i in range(4)])
        outs = [oracles[i].step(int(acts[i])) for i in range(4)]
        want = np.stack([o[0] if not o[2] else oracles[i].reset() for i, o in enumerate(outs)])
        g = env.step(acts)
        assert np.array_equal(g[0].cpu().numpy(), want.astype(np.float32)), t
    assert env.debug_state()["cursor"].max() > 5
    env.close()


def test_full_size_properties():
    """BASELINE config 1 size (4096 bins, BlockOut, R = 4): size-independent properties --
    determinism across two instances, heightmap monotone within an episode and reset to zero on done,
    observation's heightmap block equal to the float64 state, candidate rows consistent with V/padding."""
    import torch
    from irbpp_b200 import shapes
    n = 4096
    lib = shapes.make_blockout_library(32, seed=1)
    seqs = shapes.make_sequences(n, 64, lib.num_shapes, seed=0)
    a = _env(lib, seqs); b = _env(lib, seqs)
    oa = a.reset(); ob = b.reset()
    assert torch.equal(oa, ob)
    gen = torch.Generator(device="cuda:0"); gen.manual_seed(0)
    prev_hm = a.debug_state()["heightmap"]
    assert not prev_hm.any()
    total_done = 0
    for t in range(30):
        cand = oa[:, :2500].view(n, 500, 5)
        mask = cand[:, :, 4] == 1
        score = torch.rand((n, 500), device="cuda:0", generator=gen) + mask.float()
        acts = torch.argmax(score, dim=1)
        oa, ra, da, ia = a.step(acts)
        ob, rb, db, ib = b.step(acts.cpu().numpy())
        assert torch.equal(oa, ob) and torch.equal(ra, rb) and np.array_equal(da, db)
        hm = a.debug_state()["heightmap"]
        assert np.array_equal(oa[:, 2509:].cpu().numpy(), hm.reshape(n, -1).astype(np.float32))
        keep = ~da
        assert (hm[keep] >= prev_hm[keep]).all()
        assert not hm[da].any()
        assert (ra.numpy()[:, 0][da] == 0).all() and (ra.numpy()[:, 0][keep] > 0).all()
        c = oa[:, :2500].view(n, 500, 5).cpu().numpy()
        assert ((c[:, :, 4] == 0) | (c[:, :, 4] == 1)).all()
        assert (c[:, :, 0] < 4).all() and (c[:, :, 1] < 16).all() and (c[:, :, 2] < 16).all()
        assert (c[:, :, 3][c[:, :, 4] == 1] <= 0.30).all()
        prev_hm = hm
        total_done += int(da.sum())
    assert total_done > 0
    assert a.launch_count() == 62          # (scan + candidates kernel) per reset / step
    a.close(); b.close()


def test_full_size_subset_matches_oracle():
    """4096 bins on the GPU, a random subset of 40 of them replayed by the oracle with the same actions:
    bins are independent, so this is a value-exact check at the benchmark's batch size."""
    import torch
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleConfig, OracleEnv
    n = 4096
    lib = shapes.make_blockout_library(32, seed=1)
    seqs = shapes.make_sequences(n, 128, lib.num_shapes, seed=0)
    env = _env(lib, seqs)
    rng = np.random.default_rng(11)
    subset = np.sort(rng.choice(n, size=40, replace=False))
    cfg = OracleConfig(ZRotNum=4)
    oracles = [OracleEnv(cfg, lib, seqs[i]) for i in subset]
    obs = env.reset()
    want = np.stack([o.reset() for o in oracles])
    assert np.array_equal(obs[subset].cpu().numpy(), want.astype(np.float32))
    gen = torch.Generator(device="cuda:0"); gen.manual_seed(3)
    ep_r = [[] for _ in subset]
    n_done = 0
    for t in range(45):
        mask = obs[:, :2500].view(n, 500, 5)[:, :, 4] == 1
        acts = torch.argmax(torch.rand((n, 500), device="cuda:0", generator=gen) + mask.float(), dim=1)
        obs, rew, done, infos = env.step(acts)
        a = acts.cpu().numpy()
        for k, i in enumerate(subset):
            o, r, d, info = oracles[k].step(int(a[i]))
            ep_r[k].append(r)
            if d:
                gi = infos[int(i)]
                assert gi["counter"] == info["counter"] and gi["ratio"] == info["ratio"]
                assert gi["episode"]["r"] == round(sum(ep_r[k]), 6) and gi["episode"]["l"] == len(ep_r[k])
                ep_r[k] = []
                o = oracles[k].reset()
                n_done += 1
            want[k] = o
            assert np.float32(r) == rew[int(i), 0].item() and bool(d) == bool(done[i])
        assert np.array_equal(obs[subset].cpu().numpy(), want.astype(np.float32)), t
    assert n_done > 0
    env.close()


def test_c_abi_error_behaviour():
    """Error codes of the C ABI (include/irbpp.h): call order, argument validation, table validation."""
    import ctypes
    from irbpp_b200 import _lib, shapes
    lib = _lib.load()
    cfg = _lib.IrbppConfig()
    cfg.num_envs, cfg.num_rotations, cfg.selected_action, cfg.buffer_size = 4, 4, 500, 1
    cfg.bin_dimension[0], cfg.bin_dimension[1], cfg.bin_dimension[2] = 0.32, 0.32, 0.30
    cfg.resolution_act, cfg.resolution_h, cfg.resolution_z = 0.02, 0.01, 0.01
    cfg.device = 0
    h = ctypes.c_void_p()
    assert lib.irbpp_create(ctypes.byref(cfg), ctypes.byref(h)) == _lib.IRBPP_OK
    import torch
    obs = torch.empty((4, 3533), dtype=torch.float32, device="cuda:0")
    acts = np.zeros(4, dtype=np.int64)
    # nothing loaded yet
    assert lib.irbpp_reset(h, None, obs.data_ptr(), None) == _lib.IRBPP_ESTATE
    sl = shapes.make_blockout_library(6, seed=3)
    dims, ext, vol, maps, offsets = sl.flat()
    # rotation count mismatch, out-of-range table, non-0/1 mask
    assert lib.irbpp_load_shapes(h, 6, 2, dims.ctypes.data, ext.ctypes.data, vol.ctypes.data, maps.ctypes.data,
                                 offsets.ctypes.data, maps.size) == _lib.IRBPP_EINVAL
    assert lib.irbpp_load_shapes(h, 6, 4, dims.ctypes.data, ext.ctypes.data, vol.ctypes.data, maps.ctypes.data,
                                 offsets.ctypes.data, maps.size - 8) == _lib.IRBPP_EINVAL
    bad = maps.copy(); n0 = int(dims[0, 0, 0] * dims[0, 0, 1]); bad[int(offsets[0, 0]) + 3 * n0] = 0.5
    assert lib.irbpp_load_shapes(h, 6, 4, dims.ctypes.data, ext.ctypes.data, vol.ctypes.data, bad.ctypes.data,
                                 offsets.ctypes.data, maps.size) == _lib.IRBPP_EINVAL
    assert b"masks must be 0/1" in lib.irbpp_last_error(h)
    # a window wider than its action footprint: the reference's slice would run off the heightmap
    d2 = dims.copy(); d2[0, 0, 2] = 1
    assert lib.irbpp_load_shapes(h, 6, 4, d2.ctypes.data, ext.ctypes.data, vol.ctypes.data, maps.ctypes.data,
                                 offsets.ctypes.data, maps.size) == _lib.IRBPP_EINVAL
    assert lib.irbpp_load_shapes(h, 6, 4, dims.ctypes.data, ext.ctypes.data, vol.ctypes.data, maps.ctypes.data,
                                 offsets.ctypes.data, maps.size) == _lib.IRBPP_OK
    ids = np.zeros((4, 8), dtype=np.int32); ids[2, 3] = 6
    assert lib.irbpp_set_sequences(h, ids.ctypes.data, 8) == _lib.IRBPP_EINVAL            # id out of range
    ids[2, 3] = 5
    assert lib.irbpp_set_sequences(h, ids.ctypes.data, 8) == _lib.IRBPP_OK
    # call order: step before reset, wait without step, double step_async, buffered-only calls
    assert lib.irbpp_step_async(h, acts.ctypes.data, 0, obs.data_ptr(), None) == _lib.IRBPP_ESTATE
    assert lib.irbpp_step_wait(h, None) == _lib.IRBPP_ESTATE
    assert lib.irbpp_reset(h, None, obs.data_ptr(), None) == _lib.IRBPP_OK
    assert lib.irbpp_step_async(h, acts.ctypes.data, 0, obs.data_ptr(), None) == _lib.IRBPP_OK
    assert lib.irbpp_step_async(h, acts.ctypes.data, 0, obs.data_ptr(), None) == _lib.IRBPP_ESTATE
    assert b"already running" in lib.irbpp_last_error(h)
    assert lib.irbpp_step_wait(h, None) == _lib.IRBPP_OK
    assert lib.irbpp_get_action_candidates(h, acts.ctypes.data, 0, obs.data_ptr(), None) == _lib.IRBPP_ESTATE
    assert lib.irbpp_get_all_possible_observation(h, obs.data_ptr(), None) == _lib.IRBPP_ESTATE
    assert lib.irbpp_step_async(h, None, 0, obs.data_ptr(), None) == _lib.IRBPP_EINVAL
    assert lib.irbpp_launch_count(h) == 4
    assert lib.irbpp_destroy(h) == _lib.IRBPP_OK


def test_two_handles_with_different_libraries_coexist():
    """Per-function CUDA attributes are shared by all handles of the process: a small-table handle created
    after a large-table one must not break the first."""
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleConfig, OracleVecEnv
    big = shapes.make_irregular_library(8, seed=5)
    small = shapes.make_cube_library(seed=6, num_shapes=6)
    sa = shapes.make_sequences(6, 16, big.num_shapes, seed=1)
    sb = shapes.make_sequences(6, 16, small.num_shapes, seed=2)
    a = _env(big, sa)
    b = _env(small, sb)
    oa = OracleVecEnv(OracleConfig(ZRotNum=8), big, sa)
    ob = OracleVecEnv(OracleConfig(ZRotNum=2), small, sb)
    assert np.array_equal(a.reset().cpu().numpy(), oa.reset().astype(np.float32))
    assert np.array_equal(b.reset().cpu().numpy(), ob.reset().astype(np.float32))
    for t in range(6):
        acts = np.zeros(6, dtype=np.int64)
        assert np.array_equal(a.step(acts)[0].cpu().numpy(), oa.step(acts)[0].astype(np.float32))
        assert np.array_equal(b.step(acts)[0].cpu().numpy(), ob.step(acts)[0].astype(np.float32))
    a.close(); b.close()


def test_24_rotations_match_oracle():
    """BASELINE.json config 3 speaks of 24 poses per shape; the rotation count is a runtime parameter
    (up to 32).  6 rotation groups per scan CTA, 24 x levels images per bin in the candidates kernel."""
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleConfig, OracleVecEnv
    lib = shapes.make_irregular_library(6, seed=9, num_rotations=24)
    seqs = shapes.make_sequences(6, 24, lib.num_shapes, seed=4)
    ora = OracleVecEnv(OracleConfig(ZRotNum=24), lib, seqs)
    env = _env(lib, seqs)
    o = ora.reset(); g = env.reset()
    assert np.array_equal(g.cpu().numpy(), o.astype(np.float32))
    rng = np.random.default_rng(2)
    max_valid = 0
    for t in range(14):
        acts = _random_valid_actions(rng, o, 500)
        max_valid = max(max_valid, int((o[:, :2500].reshape(6, 500, 5)[:, :, 4] == 1).sum(axis=1).max()))
        o, orew, odone, _ = ora.step(acts)
        g, grew, gdone, _ = env.step(acts)
        assert np.array_equal(g.cpu().numpy(), o.astype(np.float32)), t
        assert np.array_equal(gdone, odone)
    assert max_valid == 500          # with 24 rotations the >selectedAction truncation is the normal case
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["heuristic_blockout", "heuristic_irregular"])
def test_heuristic_episode_matches_reference_golden(name):
    """irbpp_heuristic_actions + irbpp_step_poses_async against episodes generated by the reference's own
    Space.get_heuristic_action (space.py:162-227): every score x flip direction at every step, host and
    device outputs, then a pose step."""
    from irbpp_b200.vec_env import GpuVecEnv
    d = load_golden(name)
    lib = lib_from_fixture(d)
    env = _env(lib, d["sequences"])
    obs = env.reset()
    assert np.array_equal(obs.cpu().numpy(), d["obs"][0])
    for t in range(len(d["actions"])):
        for mi, m in enumerate(GpuVecEnv.HEURISTICS):
            for k in range(4):
                poses, index = env.get_heuristic_actions(m, k)
                assert np.array_equal(poses, d["poses"][t, mi, k]), (t, m, k)
                assert np.array_equal(index, d["index"][t, mi, k]), (t, m, k)
        pt, it = env.get_heuristic_actions("HM", t % 4, as_tensor=True)
        assert pt.is_cuda and np.array_equal(pt.cpu().numpy(), d["poses"][t, 3, t % 4])
        assert np.array_equal(it.cpu().numpy(), d["index"][t, 3, t % 4])
        if t % 2:
            p = d["poses"][t, t % 4, (t // 4) % 4]
            obs, rew, done, infos = env.step_poses(p)                        # [N, 3] form
        else:
            obs, rew, done, infos = env.step_poses(d["actions"][t])         # flat int64 form
        assert np.array_equal(obs.cpu().numpy(), d["obs"][t + 1]), t
        assert np.array_equal(rew.numpy()[:, 0], d["reward"][t].astype(np.float32))
        assert np.array_equal(done, d["done"][t])
    env.close()


@pytest.mark.gpu
def test_heuristic_policy_matches_oracle_at_scale():
    """96 bins stepped with the heuristic poses, the method and flip direction changing over time; CUDA path
    vs the oracle, including auto-resets; plus the call-order errors."""
    from irbpp_b200 import shapes, _lib
    from irbpp_b200.vec_env import GpuVecEnv
    from oracle.oracle_env import OracleConfig, OracleVecEnv
    lib = shapes.make_irregular_library(16, seed=41, num_rotations=4)
    seqs = shapes.make_sequences(96, 64, lib.num_shapes, seed=8)
    ora = OracleVecEnv(OracleConfig(ZRotNum=4), lib, seqs)
    env = _env(lib, seqs)
    o = ora.reset(); g = env.reset()
    ndone = 0
    for t in range(60):
        m = GpuVecEnv.HEURISTICS[(t // 5) % 4]
        po, io = ora.heuristic_actions(m, t % 4)
        pg, ig = env.get_heuristic_actions(m, t % 4)
        assert np.array_equal(pg, po) and np.array_equal(ig, io), (t, m)
        flat = (po[:, 0].astype(np.int64) * 16 + po[:, 1]) * 16 + po[:, 2]
        o, orew, odone, _ = ora.step(flat, poses=True)
        g, grew, gdone, _ = env.step_poses(flat)
        assert np.array_equal(g.cpu().numpy(), o.astype(np.float32)), t
        assert np.array_equal(gdone, odone)
        ndone += int(odone.sum())
    assert ndone > 0
    # an out-of-range pose is a device error like an out-of-range candidate row
    bad = np.full(96, 4 * 256, dtype=np.int64)
    with pytest.raises(RuntimeError):
        env.step_poses(bad)
    with pytest.raises(ValueError):
        env.get_heuristic_actions("RANDOM")
    env.close()
    # buffered mode: heuristics need get_action_candidates first
    seqs2 = shapes.make_sequences(8, 32, lib.num_shapes, seed=9)
    envb = _env(lib, seqs2, buffer_size=3)
    envb.reset()
    with pytest.raises(RuntimeError):
        envb.get_heuristic_actions("MINZ")
    envb.get_action_candidates(np.zeros(8, dtype=np.int64))
    orab = OracleVecEnv(OracleConfig(ZRotNum=4, bufferSize=3), lib, seqs2)
    orab.reset(); orab.get_action_candidates(np.zeros(8, dtype=np.int64))
    pg, ig = envb.get_heuristic_actions("DBLF", 1)
    po, io = orab.heuristic_actions("DBLF", 1)
    assert np.array_equal(pg, po) and np.array_equal(ig, io)
    envb.close()


@pytest.mark.gpu
def test_survey_known_answers_on_device():
    """SURVEY.md section 4: the known-answer level sets of the unmodified cvTools (rectangle, pixel, line, L
    with a collapsing notch, ring + island, diagonals, the two-level map) through irbpp_debug_hulls."""
    from irbpp_b200 import shapes
    from test_kernels_emulated import check_kats
    env = _env(shapes.make_cube_library(seed=1, num_rotations=1, num_shapes=4), _dummy_seqs(8, None), selected_action=256)

    def run(pv, mk):
        out = env.debug_hulls(pv, mk)
        return out["cand"], out["num_hull"]
    check_kats(run)
    env.close()


@pytest.mark.gpu
def test_many_start_pixels_on_device():
    """More start pixels in a round than the task table lists (search fallback, several batches)."""
    from irbpp_b200 import shapes
    from test_kernels_emulated import check_many_start_pixels
    env = _env(shapes.make_cube_library(seed=1, num_rotations=1, num_shapes=4), _dummy_seqs(4, None), selected_action=256)

    def run(pv, mk):
        out = env.debug_hulls(pv, mk)
        return out["cand"], out["num_hull"]
    check_many_start_pixels(run)
    env.close()
