"""The 32 x 32 action grid (resolutionA = resolutionH = 0.01, stepSize 1: what the reference trains the Cube dataset
with) without a GPU: configuration checks of the product library, the cv2-free contour port on 32 x 32 images, and the
kernels' Grid<1> instantiations on host threads (tests/host_harness/cuda_emu.h) against the oracle at resolutionAct 0.01."""
import ctypes

import numpy as np
import pytest

from irbpp_b200 import _lib, shapes
from oracle import contours_port
from oracle.oracle_env import (OracleConfig, OracleEnv, OracleVecEnv, convex_hull_actions, heuristic_action_port,
                               scan_vectorized)
from test_kernels_emulated import EmuEnv, build_emulated, _P

pytestmark = pytest.mark.timeout(900)          # a deadlocked emulated barrier must not hang the suite

RES_A = 0.01
A = 32                                         # actions per axis


@pytest.fixture(scope="module")
def built_lib():
    from irbpp_b200 import build
    return build.build()


def _config(n=4, R=2, sel=500, k=1, res_act=RES_A):
    return _lib.IrbppConfig(n, R, sel, k, (ctypes.c_double * 3)(0.32, 0.32, 0.30), res_act, 0.01, 0.01, 0, 0)


def test_create_accepts_fine_grid_without_gpu(built_lib):
    """A stepSize-1 configuration passes validation and stops at the device query (no CPU path); other grids are still
    rejected, naming both supported ones; the pose count of the selected_action check is the grid's own (R * 1024)."""
    import torch
    lib = _lib.load()
    h = ctypes.c_void_p()
    for bad in (0.04, 0.015):                  # stepSize 4, and a non-integer stepSize
        cfg = _config(res_act=bad)
        assert lib.irbpp_create(ctypes.byref(cfg), ctypes.byref(h)) == _lib.IRBPP_EINVAL
        msg = lib.irbpp_last_error(None)
        assert b"unsupported grid" in msg and b"16x16" in msg and b"32x32" in msg, msg
    cfg = _config(R=2, sel=2049)               # more rows than the 2 * 1024 poses
    assert lib.irbpp_create(ctypes.byref(cfg), ctypes.byref(h)) == _lib.IRBPP_EINVAL
    if torch.cuda.is_available():
        pytest.skip("GPU present: creation succeeds there (tests/test_gpu_fine_grid.py)")
    cfg = _config(R=2, sel=2048)               # would be rejected on the 16x16 grid (512 poses)
    assert lib.irbpp_create(ctypes.byref(cfg), ctypes.byref(h)) == _lib.IRBPP_ECUDA
    assert b"no CPU path" in lib.irbpp_last_error(None)


def _rand_level_map(rng, kind):
    """posZValid / mask of one 32 x 32 rotation: random plateaus, sparse noise, or long borders."""
    pv = np.full((A, A), 1e3)
    mk = np.zeros((A, A))
    xs, ys = np.meshgrid(np.arange(A), np.arange(A), indexing="ij")
    if kind == 0:                              # plateaus of a few levels
        mk[:] = rng.random((A, A)) < 0.9
        pv[:] = 0.01 * rng.integers(0, 4, size=(A, A)) + 0.005
        for _ in range(int(rng.integers(2, 8))):
            x0, y0 = rng.integers(0, A - 4, 2); w, h = rng.integers(2, 14, 2)
            pv[x0:x0 + w, y0:y0 + h] = 0.01 * int(rng.integers(0, 5)) + 0.005
    elif kind == 1:                            # sparse noise
        mk[:] = rng.random((A, A)) < rng.uniform(0.2, 0.7)
        pv[:] = 0.005
    else:                                      # one ragged component with a long border (many overflow redos)
        mk[:] = 1
        pv[:] = 0.015
        rag = (xs % 2 == 0) | (rng.random((A, A)) < 0.3)
        pv[~rag] = 0.035
    pv[mk == 0] = 1e3
    return pv, mk


def test_contour_port_matches_cv2_32x32():
    """oracle/contours_port.py against the cv2 restatement of cvTools.convexHulls on 32 x 32 maps (random, noisy and
    long-border images), i.e. the oracle the kernel tests below rely on is right at this size."""
    pytest.importorskip("cv2")
    from oracle.oracle_env import convex_hulls_cv2
    rng = np.random.default_rng(11)
    n = 0
    for i in range(120):
        pv, mk = _rand_level_map(rng, i % 3)
        got, gv = contours_port.convex_hulls_port(pv, mk, 0.01)
        want, wv = convex_hulls_cv2(pv, mk, 0.01)
        assert np.array_equal(np.asarray(got), np.asarray(want)), i
        if len(want):
            assert np.array_equal(gv, wv), i
            n += len(want)
    assert n > 1000


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emulated(str(tmp_path_factory.mktemp("emu_fine")))


class FineEmuEnv(EmuEnv):
    """EmuEnv at resolutionAct 0.01."""

    def __init__(self, lib, library, sequences, selected_action=500, buffer_size=1):
        self.lib, self.n = lib, len(sequences)
        cfg = _config(self.n, library.num_rotations, selected_action, buffer_size)
        self.h = ctypes.c_void_p()
        assert lib.emu_irbpp_create(ctypes.byref(cfg), ctypes.byref(self.h)) == 0
        dims, ext, vol, maps, offsets = library.flat()
        P = ctypes.c_void_p
        assert lib.emu_irbpp_load_shapes(self.h, library.num_shapes, library.num_rotations, P(dims.ctypes.data),
                                         P(ext.ctypes.data), P(vol.ctypes.data), P(maps.ctypes.data),
                                         P(offsets.ctypes.data), ctypes.c_int64(maps.size)) == 0
        seqs = np.ascontiguousarray(sequences, dtype=np.int32)
        assert lib.emu_irbpp_set_sequences(self.h, P(seqs.ctypes.data), seqs.shape[1]) == 0
        o, l, k = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
        lib.emu_irbpp_obs_len(self.h, ctypes.byref(o), ctypes.byref(l), ctypes.byref(k))
        self.obs_len, self.loc_len = o.value, l.value


def _random_valid(rng, rows, sel):
    valid = np.nonzero(rows[:sel * 5].reshape(sel, 5)[:, 4] == 1)[0]
    return int(rng.choice(valid)) if len(valid) else 0


def _play(emu, lib, sel, steps, n=3, k=1, seed=0):
    """Online (k = 1) or buffered episodes, random valid actions, against OracleVecEnv; returns (dones, truncated rows)."""
    R = lib.num_rotations
    seqs = shapes.make_sequences(n, 64, lib.num_shapes, seed=seed)
    ora = OracleVecEnv(OracleConfig(resolutionAct=RES_A, ZRotNum=R, selectedAction=sel, bufferSize=k), lib, seqs)
    env = FineEmuEnv(emu, lib, seqs, selected_action=sel, buffer_size=k)
    want = ora.reset()
    obs = env.reset()
    assert np.array_equal(obs, want.astype(np.float32))
    rng = np.random.default_rng(seed)
    dones = trunc = 0
    for t in range(steps):
        if k > 1:
            all_o = np.stack([e.get_all_possible_observation() for e in ora.envs])
            assert np.array_equal(env.get_all_possible_observation(k), all_o.astype(np.float32)), t
            order = rng.integers(0, k, size=n)
            loc = np.stack(ora.get_action_candidates(order))
            assert np.array_equal(env.get_action_candidates(order), loc.astype(np.float32)), t
        else:
            loc = want
        trunc += int((loc[:, (sel - 1) * 5:(sel - 1) * 5 + 3].sum(1) > 0).sum())
        acts = np.array([_random_valid(rng, loc[i], sel) for i in range(n)], dtype=np.int64)
        want, rew, done, infos = ora.step(acts)
        obs, res = env.step_results(acts)
        assert np.array_equal(obs, want.astype(np.float32)), t
        assert np.array_equal(res["reward"], rew.astype(np.float32)) and np.array_equal(res["done"].astype(bool), done), t
        assert not res["error"].any(), t
        for i in np.nonzero(done)[0]:
            assert res["counter"][i] == infos[i]["counter"] and res["ratio"][i] == infos[i]["ratio"], (t, i)
        dones += int(done.sum())
    env.close()
    return dones, trunc


def test_emulated_fine_cube_episodes(emu):
    """Cube items (R = 2) on the 32 x 32 grid: full float32 observations, reward / done / counter / ratio and the
    auto-resets of the episodes that end."""
    lib = shapes.make_cube_library(seed=3, num_rotations=2, resolutionAct=RES_A)
    dones, _ = _play(emu, lib, 500, 16, seed=1)
    assert dones > 0


def test_emulated_fine_blockout_truncation(emu):
    """BlockOut shapes (R = 4) at resolutionAct 0.01 with a table far smaller than the candidate set: every step takes
    the bucketed truncation ranking of phase D over R * 1024 poses, and the scan runs the per-cell lists (no block
    form at stepSize 1)."""
    lib = shapes.make_blockout_library(10, seed=4, resolutionAct=RES_A)
    dones, trunc = _play(emu, lib, 40, 12, seed=2)
    assert trunc > 0


def test_emulated_fine_buffered_protocol(emu):
    """Buffered episodes (k = 5): get_all_possible_observation (one scan per buffered item), get_action_candidates and
    the order observations of the steps."""
    lib = shapes.make_cube_library(seed=5, num_rotations=2, resolutionAct=RES_A)
    _play(emu, lib, 200, 4, n=2, k=5, seed=3)


def test_emulated_fine_scan_and_heuristics(emu):
    """irbpp_debug_scan on random heightmaps against the scan restatement, then the four heuristics in all four
    directions and a step with the chosen poses, against the oracle."""
    lib = shapes.make_irregular_library(6, seed=7, num_rotations=2, resolutionAct=RES_A)
    n, R = 3, 2
    seqs = shapes.make_sequences(n, 32, lib.num_shapes, seed=4)
    cfg = OracleConfig(resolutionAct=RES_A, ZRotNum=R)
    env = FineEmuEnv(emu, lib, seqs)
    rng = np.random.default_rng(9)
    hm = np.round(rng.random((n, 32, 32)) * 0.08, 3)
    hm[0] = 0.0
    env.reset()
    assert emu.emu_irbpp_debug_set_heightmap(env.h, _P(np.ascontiguousarray(hm))) == 0
    items = np.array([0, 3, 5], np.int32)
    pz, pv, mk = (np.zeros((n, R, A, A)) for _ in range(3))
    cand, nh = np.zeros((n, 500, 5)), np.zeros(n, np.int32)
    assert emu.emu_irbpp_debug_scan(env.h, _P(items), _P(pz), _P(pv), _P(mk), _P(cand), _P(nh)) == 0
    for i in range(n):
        wz, wv, wm = scan_vectorized(cfg, hm[i], lib.extents[items[i]], lib.tables[items[i]])
        assert np.array_equal(pz[i], wz) and np.array_equal(pv[i], wv) and np.array_equal(mk[i], wm), i
        hull = convex_hull_actions(wv, wm, 0.01, "port")
        assert nh[i] == (0 if hull is None else len(hull)), i
    env.close()

    env = FineEmuEnv(emu, lib, seqs)
    oracles = [OracleEnv(cfg, lib, seqs[i]) for i in range(n)]
    want = np.stack([o.reset() for o in oracles])
    assert np.array_equal(env.reset(), want.astype(np.float32))
    for t in range(3):
        for mi, method in enumerate(("MINZ", "DBLF", "FIRSTFIT", "HM")):
            for d in range(4):
                poses, index = np.zeros((n, 3), np.int32), np.zeros(n, np.int64)
                assert emu.emu_irbpp_heuristic_actions(env.h, mi, d, _P(poses), _P(index), 0, None) == 0
                for i, o in enumerate(oracles):
                    wp = heuristic_action_port(cfg, lib, o.heightmap, o.next_item_ID, o.posZmap, o.naiveMask, method, d)
                    assert tuple(poses[i]) == tuple(wp) and index[i] == o.candidate_index(wp), (t, method, d, i)
        poses, _ = np.zeros((n, 3), np.int32), None
        assert emu.emu_irbpp_heuristic_actions(env.h, t % 4, 0, _P(poses), _P(np.zeros(n, np.int64)), 0, None) == 0
        flat = np.ascontiguousarray((poses[:, 0].astype(np.int64) * A + poses[:, 1]) * A + poses[:, 2])
        obs = np.zeros((n, env.obs_len), np.float32)
        assert emu.emu_irbpp_step_poses_async(env.h, _P(flat), 0, _P(obs), None) == 0
        assert emu.emu_irbpp_step_wait(env.h, None) == 0
        for i, o in enumerate(oracles):
            w, _, d, _ = o.step_pose(*[int(v) for v in poses[i]])
            want[i] = o.reset() if d else w
        assert np.array_equal(obs, want.astype(np.float32)), t
    env.close()


def test_emulated_fine_hulls_and_overflow(emu):
    """irbpp_debug_hulls on 32 x 32 maps against the contour port: random maps, and a maximal-border image (an
    8-connected checkerboard: one component whose border passes most pixels several times), which takes the serial
    overflow redo with the global 4096-point buffer and must not report IRBPP_EDEVICE code 6."""
    lib = shapes.make_cube_library(seed=1, num_rotations=1, num_shapes=4, resolutionAct=RES_A)
    rng = np.random.default_rng(3)
    maps = [_rand_level_map(rng, i % 3) for i in range(6)]
    xs, ys = np.meshgrid(np.arange(A), np.arange(A), indexing="ij")
    checker = ((xs + ys) % 2 == 0).astype(np.float64)
    maps.append((np.where(checker == 1, 0.005, 1e3), checker))
    n = len(maps)
    env = FineEmuEnv(emu, lib, np.zeros((n, 8), np.int32), selected_action=1024)
    pv = np.ascontiguousarray(np.stack([m[0] for m in maps])[:, None])
    mk = np.ascontiguousarray(np.stack([m[1] for m in maps])[:, None])
    cand, nh = np.zeros((n, 1024, 5)), np.zeros(n, np.int32)
    counters = np.zeros(8, np.uint64)
    assert emu.emu_irbpp_debug_phase_cycles(env.h, 1, _P(counters)) == 0
    assert emu.emu_irbpp_debug_hulls(env.h, _P(pv), _P(mk), _P(cand), _P(nh)) == 0, emu.emu_irbpp_last_error(env.h)
    assert emu.emu_irbpp_debug_phase_cycles(env.h, 0, _P(counters)) == 0
    assert counters[7] > 0                     # overflow redos ran
    for i in range(n):
        want = convex_hull_actions(pv[i], mk[i], 0.01, "port")
        assert want is not None and nh[i] == len(want), i
        k = min(len(want), 1024)
        assert np.array_equal(cand[i, :k], want[:k]), i
    env.close()


def test_gpu_vec_env_checks_resolution_act_against_library():
    """GpuVecEnv takes the action resolution from the library; a caller value that differs is refused before any
    device work (a library built for one grid scanned with the windows of another would be silently wrong)."""
    from irbpp_b200.vec_env import GpuVecEnv
    lib = shapes.make_cube_library(seed=1, num_rotations=2, num_shapes=4, resolutionAct=RES_A)
    with pytest.raises(ValueError, match="resolutionAct"):
        GpuVecEnv(lib, np.zeros((2, 4), np.int32), resolution_act=0.02)
    lib2 = shapes.make_cube_library(seed=1, num_rotations=2, num_shapes=4)
    with pytest.raises(ValueError, match="resolutionAct"):
        GpuVecEnv(lib2, np.zeros((2, 4), np.int32), resolution_act=RES_A)


def test_emulated_packed_observations_round_trip_fine(emu):
    """The compact form of the rollout gather (csrc/irbpp_pack.cuh) is lossless on the 32 x 32 grid: poses with
    x, y up to 31 and rotations up to 31 -- a fine-grid reset observation and a synthetic one with every extreme."""
    lib = shapes.make_cube_library(seed=3, num_rotations=2, resolutionAct=RES_A)
    seqs = shapes.make_sequences(2, 8, lib.num_shapes, seed=1)
    env = FineEmuEnv(emu, lib, seqs)
    obs = env.reset()
    env.close()
    sel = 500
    rows = obs[:, :sel * 5].reshape(2, sel, 5)
    assert rows[:, :, 1:3].max() > 15
    rng = np.random.default_rng(0)
    synth = obs.copy()
    srows = synth[:, :sel * 5].reshape(2, sel, 5)
    srows[:, :, 0] = rng.integers(0, 32, size=(2, sel))
    srows[:, :, 1:3] = rng.integers(0, 32, size=(2, sel, 2))
    srows[:, -1, :3] = 31
    synth = np.ascontiguousarray(synth)
    for o in (np.ascontiguousarray(obs), synth):
        n, width = o.shape
        packed = np.zeros((n, emu.emu_irbpp_packed_obs_bytes(sel)), np.uint8)
        assert emu.emu_irbpp_pack_observations(_P(o), ctypes.c_int64(width), sel, n, _P(packed), None) == 0
        back = np.full((n, width), -7.0, np.float32)
        assert emu.emu_irbpp_unpack_observations(_P(packed), sel, n, _P(back), ctypes.c_int64(width), None) == 0
        assert np.array_equal(back, o)


_ASAN_CHILD = r'''
import sys, tempfile
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import test_fine_grid as f
from test_kernels_emulated import build_emulated
emu = build_emulated(tempfile.mkdtemp(), defs=["-fsanitize=address", "-g", "-fno-omit-frame-pointer"])
f.check_hulls_partial_cta(emu)
print("asan child ok")
'''


def check_hulls_partial_cta(emu):
    """irbpp_debug_hulls on 3 bins (R = 1: 4-bin CTAs, so the last CTA has an idle warp) of long-border 32 x 32 maps:
    the idle warp's lanes take contour tasks too, and their overflow redos need buffers of their own."""
    lib = shapes.make_cube_library(seed=1, num_rotations=1, num_shapes=4, resolutionAct=RES_A)
    rng = np.random.default_rng(5)
    maps = [_rand_level_map(rng, 2) for _ in range(2)]
    xs, ys = np.meshgrid(np.arange(A), np.arange(A), indexing="ij")
    checker = ((xs + ys) % 2 == 0).astype(np.float64)
    maps.append((np.where(checker == 1, 0.005, 1e3), checker))
    n = len(maps)
    env = FineEmuEnv(emu, lib, np.zeros((n, 8), np.int32), selected_action=1024)
    pv = np.ascontiguousarray(np.stack([m[0] for m in maps])[:, None])
    mk = np.ascontiguousarray(np.stack([m[1] for m in maps])[:, None])
    cand, nh = np.zeros((n, 1024, 5)), np.zeros(n, np.int32)
    counters = np.zeros(8, np.uint64)
    assert emu.emu_irbpp_debug_phase_cycles(env.h, 1, _P(counters)) == 0
    assert emu.emu_irbpp_debug_hulls(env.h, _P(pv), _P(mk), _P(cand), _P(nh)) == 0
    assert emu.emu_irbpp_debug_phase_cycles(env.h, 0, _P(counters)) == 0
    assert counters[7] > 0                     # overflow redos ran
    for i in range(n):
        want = convex_hull_actions(pv[i], mk[i], 0.01, "port")
        assert nh[i] == len(want) and np.array_equal(cand[i, :len(want)], want), i
    env.close()


def test_emulated_fine_overflow_buffers_of_a_partial_cta_under_asan():
    """The kernels under AddressSanitizer (host emulator, child process): a bin count that is not a multiple of the
    bins per candidates CTA, with contours long enough for the overflow redo, must stay inside every allocation."""
    import os
    import subprocess
    import sys
    libasan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(libasan):
        pytest.skip("no libasan")
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, LD_PRELOAD=libasan, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-c", _ASAN_CHILD, here, os.path.dirname(here)], capture_output=True,
                       text=True, env=env, timeout=800)
    assert r.returncode == 0 and "asan child ok" in r.stdout and "AddressSanitizer" not in r.stderr, r.stderr[-3000:]
