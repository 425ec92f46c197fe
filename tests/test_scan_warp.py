"""The one-warp-per-bin scan kernel (irbpp_scan_warp_kernel), which runs the online step of every library whose bottom
tables are all in block form (BlockOut) on the 16x16 action grid, against the CPU oracle: episodes through their
auto-resets on both block sizes, invalid actions (error code 2, auto-reset) and bin counts that leave the last CTA of four
bins partly empty.  Under the host emulation, and on the GPU when one is present.  Trajectory replay until every bin is
idle runs through this kernel in test_item_sources.py (BlockOut, buffer size 1, six bins: a CTA of four and one of two)."""
import ctypes

import numpy as np
import pytest

from oracle.oracle_env import OracleConfig, OracleEnv
from test_item_sources import EDEVICE, first_valid
from test_kernels_emulated import EmuEnv, build_emulated

SEL = 500

pytestmark = pytest.mark.timeout(1800)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emulated(str(tmp_path_factory.mktemp("emu_scan_warp")))


def _library(edge, shapes_n=12, seed=3):
    from irbpp_b200 import shapes
    return shapes.make_blockout_library(shapes_n, seed=seed, edge=edge)


def oracle_step(env, a):
    """One oracle step with the library's handling of an action outside the candidate table: the bin fails (done,
    counter and ratio of the episode) and auto-resets.  -> (obs, reward, done, counter, ratio, error code)"""
    if a < 0 or a >= SEL:
        counter, ratio = len(env.packed_ids), env.get_ratio()
        return env.reset(), 0.0, True, counter, ratio, 2
    o, r, d, info = env.step(int(a))
    if d:
        o = env.reset()
        return o, r, True, info["counter"], info["ratio"], 0
    return o, r, False, None, None, 0


class _Run(object):
    """Oracle envs for the bins in `check` of an N-bin run; the bins' actions: the first valid candidate of the oracle's
    observation, replaced by `bad[e]` where given."""

    def __init__(self, lib, seqs, check):
        self.check = list(check)
        self.envs = {e: OracleEnv(OracleConfig(ZRotNum=lib.num_rotations), lib, seqs[e]) for e in self.check}
        self.obs = {e: self.envs[e].reset() for e in self.check}
        self.dones = 0

    def actions(self, n, fallback_obs, bad=None):
        acts = np.array([first_valid(fallback_obs[e]) for e in range(n)], np.int64)
        for e in self.check:
            acts[e] = first_valid(self.obs[e])
        for e, a in (bad or {}).items():
            acts[e] = a
        return acts

    def step_and_compare(self, t, acts, obs, res):
        for e in self.check:
            o, r, d, counter, ratio, err = oracle_step(self.envs[e], acts[e])
            self.obs[e] = o
            assert np.array_equal(obs[e], o.astype(np.float32)), (t, e)
            assert res["reward"][e] == np.float32(r) and bool(res["done"][e]) == d and res["error"][e] == err, (t, e)
            if d:
                self.dones += 1
                assert res["counter"][e] == counter and res["ratio"][e] == ratio, (t, e)


def _emu_step(env, acts):
    """EmuEnv step that also accepts a device error: -> (rc, obs, result arrays)"""
    from irbpp_b200 import _lib
    acts = np.ascontiguousarray(acts, dtype=np.int64)
    obs = np.zeros((env.n, env.obs_len), np.float32)
    assert env.lib.emu_irbpp_step_async(env.h, ctypes.c_void_p(acts.ctypes.data), 0, ctypes.c_void_p(obs.ctypes.data), None) == 0
    res = _lib.IrbppStepResult()
    rc = env.lib.emu_irbpp_step_wait(env.h, ctypes.byref(res))
    return rc, obs, {k: np.frombuffer((ctypes.c_uint8 * (env.n * dt.itemsize)).from_address(getattr(res, k)), dtype=dt).copy()
                     for k, dt in _lib.RESULT_FIELDS}


@pytest.mark.parametrize("edge,steps", [(0.08, 14), (0.02, 3)])      # 4x4 blocks through auto-resets; 2x2 blocks
def test_emulated_warp_scan_episodes_and_invalid_actions(emu, edge, steps):
    """5 bins (a CTA of four and one of a single bin); at step 2 bins 1 and 4 send actions outside the table."""
    from irbpp_b200 import shapes
    lib = _library(edge)
    n = 5
    seqs = shapes.make_sequences(n, 64, lib.num_shapes, seed=4)
    env = EmuEnv(emu, lib, seqs)
    run = _Run(lib, seqs, range(n))
    obs = env.reset()
    for e in range(n):
        assert np.array_equal(obs[e], run.obs[e].astype(np.float32))
    for t in range(steps):
        acts = run.actions(n, obs, {1: -1, 4: SEL} if t == 2 else None)
        rc, obs, res = _emu_step(env, acts)
        assert rc == (EDEVICE if t == 2 else 0), t
        run.step_and_compare(t, acts, obs, res)
    assert run.dones >= (2 + 2 * (edge >= 0.08))
    env.close()


@pytest.mark.gpu
def test_gpu_warp_scan_4097_bins():
    """The bench's shape of step (device actions, step_device) on 4097 bins, the last CTA holding one bin; the bins of the
    first CTAs, around the middle and of the last two CTAs are checked against the oracle through auto-resets, with
    invalid actions at step 3."""
    import torch
    from irbpp_b200 import shapes
    from irbpp_b200.vec_env import GpuVecEnv
    lib = _library(0.08, 16, seed=1)
    n = 4097
    seqs = shapes.make_sequences(n, 64, lib.num_shapes, seed=0)
    check = [0, 1, 2, 3, 4, 5, 2047, 2048, 4091, 4092, 4093, 4094, 4095, 4096]
    env = GpuVecEnv(lib, seqs, device="cuda:0", selected_action=SEL)
    run = _Run(lib, seqs, check)
    obs = env.reset().cpu().numpy()
    for e in check:
        assert np.array_equal(obs[e], run.obs[e].astype(np.float32))
    for t in range(12):
        acts = run.actions(n, obs, {1: -1, 4096: SEL, 2048: 7 * SEL} if t == 3 else None)
        o, _ = env.step_device(torch.from_numpy(acts).cuda())
        res = {k: v.cpu().numpy() for k, v in env.last_step_device().items()}
        obs = o.cpu().numpy()
        run.step_and_compare(t, acts, obs, res)
        assert (res["error"] != 0).sum() == (3 if t == 3 else 0), t
    assert run.dones >= 6
    env.close()
