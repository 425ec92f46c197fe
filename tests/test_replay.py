"""The prioritized n-step replay (``memory.py``) without a GPU: ``oracle/replay_port.py`` and the device kernels of
``csrc/irbpp_replay.cuh`` under the host emulator (``test_kernels_emulated.build_emulated``) replay the fixture of the
unmodified reference (``tests/golden/replay.npz``); the bound on the stratified draws; argument validation."""
import ctypes

import numpy as np
import pytest

import replay_checks as rc
from oracle.replay_port import ReplayPort, replay_uniforms, ERR_STARVED

pytestmark = pytest.mark.timeout(900)

P = ctypes.c_void_p


def ptr(a):
    return P(a.ctypes.data)


@pytest.fixture(scope="module")
def fixture():
    return rc.load()


@pytest.mark.parametrize("bank", ["a", "b"])
def test_port_reproduces_reference(fixture, bank):
    """Trees, indices, max, t, tree indices, states, actions, nonterminals exact; R and the weights within the
    tolerance of check_bank (torch's matmul and float32 pow against a sequential sum and a correctly rounded pow)."""
    rc.check_bank(fixture, bank, rc.PortBackend(fixture, bank))


def test_port_returns_and_weights_tolerance_is_tight(fixture):
    """The stated tolerances are not slack: R of the fixture is reproduced exactly, the weights within 1 ulp."""
    d = fixture
    port = rc.PortBackend(d, "a")
    worst_r = worst_w = 0
    M, C, L, steps, rounds = rc.config(d, "a")
    r = 0
    for s in range(steps):
        port.append(d["a_app_state"][s], d["a_app_action"][s], d["a_app_reward"][s], d["a_app_done"][s],
                    d["a_app_valid"][s], float(d["a_clip"]))
        q = "ar%d_" % r
        if r < rounds and int(d[q + "step"]) == s:
            out = port.sample(np.arange(M, dtype=np.int32), int(d[q + "k"]), d[q + "uniforms"], float(d[q + "beta"]))
            worst_r = max(worst_r, rc.ulp_diff(out["returns"], d[q + "returns"]).max())
            worst_w = max(worst_w, rc.ulp_diff(out["weights"], d[q + "weights"]).max())
            port.update(d[q + "upd_mem"], d[q + "upd_idx"], d[q + "upd_loss"])
            r += 1
    assert worst_r == 0 and worst_w <= 1, (worst_r, worst_w)


def starved_port():
    """The probed hang of the reference: C = 16, twelve appends, n = 3, sample(4) -- stratum 3 is [9, 12), which holds
    only leaves 9-11, all within n of the write index (``memory.py:163-170`` would loop forever)."""
    port = ReplayPort(1, 16, 5, multi_step=3)
    for k in range(12):
        port.append(np.full((1, 5), float(k), np.float32), [k % 4], [0.5 * k], [k % 5 == 4])
    return port


def test_port_bounds_starved_stratum():
    port = starved_port()
    out = port.sample([0], 4, replay_uniforms(7, 0, 4, 64))
    assert list(out["error"]) == [0, 0, 0, ERR_STARVED]
    assert out["attempts"][3] == 64 and out["tree_idx"][3] == -1


# ---- the kernels under the host emulator -----------------------------------------------------------------------

class EmuBackend(object):
    """The replay C ABI of the emulated library driven with NumPy buffers (device == host)."""

    def __init__(self, lib, M, C, L, discount=0.99, n=3, omega=0.5):
        from irbpp_b200 import _lib
        self.lib, self.M, self.C, self.L, self.discount, self.n, self.omega = lib, M, C, L, discount, n, omega
        self.a = dict(states=np.zeros((M, C, L), np.float32), timesteps=np.zeros((M, C), np.int32),
                      actions=np.zeros((M, C), np.int64), rewards=np.zeros((M, C), np.float32),
                      nonterminals=np.zeros((M, C), np.uint8), tree=np.full((M, 2 * C - 1), np.nan, np.float32),
                      state=np.zeros((M, 4), np.int32))
        self.mem = _lib.IrbppReplayMemory(M, C, L, *(ptr(self.a[k]) for k in
                                                      ("states", "timesteps", "actions", "rewards", "nonterminals",
                                                       "tree", "state")))
        self.batch_cls = _lib.IrbppReplayBatch
        self.flags = np.zeros(1, np.uint32)
        assert lib.emu_irbpp_replay_init(ctypes.byref(self.mem), None) == 0

    def append(self, state, action, reward, done, valid, clip):
        obs = np.ascontiguousarray(np.pad(np.asarray(state, np.float32), ((0, 0), (0, 3))))   # a wider row stride
        act, rew = np.ascontiguousarray(action, np.int64), np.ascontiguousarray(reward, np.float32)
        dn, vl = np.ascontiguousarray(done, np.uint8), np.ascontiguousarray(valid, np.uint8)
        assert self.lib.emu_irbpp_replay_append(ctypes.byref(self.mem), ptr(obs), ctypes.c_int64(obs.shape[1]), ptr(act),
                                                ptr(rew), ptr(dn), ptr(vl), ctypes.c_float(clip), None) == 0

    def sample(self, mem_ids, k, uniforms, beta, seed=0, call=0, attempts=None):
        mem_ids = np.ascontiguousarray(mem_ids, np.int32)
        B, L = len(mem_ids) * k, self.L
        o = dict(tree_idx=np.zeros(B, np.int64), states=np.full((B, L), np.nan, np.float32), actions=np.zeros(B, np.int64),
                 returns=np.zeros(B, np.float32), next_states=np.full((B, L), np.nan, np.float32),
                 nonterminals=np.zeros(B, np.float32), weights=np.zeros(B, np.float32), attempts=np.zeros(B, np.int32),
                 error=np.zeros(B, np.int32))
        batch = self.batch_cls(*(ptr(o[k_]) for k_ in ("tree_idx", "states", "actions", "returns", "next_states",
                                                       "nonterminals", "weights", "attempts", "error")))
        U = None if uniforms is None else np.ascontiguousarray(uniforms, np.float64)
        A = attempts if U is None else U.shape[1]
        rc_ = self.lib.emu_irbpp_replay_sample(ctypes.byref(self.mem), ptr(mem_ids), len(mem_ids), k, self.n,
                                               ctypes.c_double(self.discount), ctypes.c_double(beta), A,
                                               ctypes.c_uint64(seed), ctypes.c_uint64(call),
                                               ptr(U) if U is not None else None, ctypes.byref(batch), ptr(self.flags), None)
        assert rc_ == 0
        return o

    def update(self, mem_ids, tree_idxs, loss):
        m, i, l_ = (np.ascontiguousarray(mem_ids, np.int32), np.ascontiguousarray(tree_idxs, np.int64),
                    np.ascontiguousarray(loss, np.float32))
        assert self.lib.emu_irbpp_replay_update_priorities(ctypes.byref(self.mem), ptr(m), ptr(i), ptr(l_), len(m),
                                                           ctypes.c_double(self.omega), ptr(self.flags), None) == 0

    def snapshot(self):
        st = self.a["state"]
        return self.a["tree"].copy(), st[:, 0].copy(), st[:, 1].copy(), st[:, 2].copy(), st[:, 3].view(np.float32).copy()


@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    from test_kernels_emulated import build_emulated
    lib = build_emulated(str(tmp_path_factory.mktemp("emu_replay")))
    lib.emu_irbpp_last_error.restype = ctypes.c_char_p
    return lib


@pytest.mark.parametrize("bank", ["a", "b"])
def test_emulated_kernels_reproduce_reference(fixture, emu_lib, bank):
    M, C, L, _, _ = rc.config(fixture, bank)
    be = EmuBackend(emu_lib, M, C, L, float(fixture["discount"]), int(fixture["n"]), float(fixture["omega"]))
    rc.check_bank(fixture, bank, be)
    assert be.flags[0] == 0


def test_emulated_kernels_match_port_with_generated_uniforms(emu_lib):
    """The counter-based uniforms (no array supplied) against their NumPy mirror, with invalid appends, terminals,
    wrap-around, k = 5 strata and duplicated / out-of-range update rows."""
    rng = np.random.default_rng(4)
    M, C, L = 4, 13, 6
    be, port = EmuBackend(emu_lib, M, C, L, n=2, omega=0.6), ReplayPort(M, C, L, multi_step=2, priority_exponent=0.6)
    expect = 0
    for step in range(40):
        args = (rng.standard_normal((M, L)).astype(np.float32), rng.integers(0, 9, M),
                rng.standard_normal(M).astype(np.float32) * 3, rng.random(M) < 0.2, rng.random(M) < 0.8, 2.0)
        be.append(*args); port.append(*args[:5], reward_clip=2.0)
        if step >= 15 and step % 3 == 0:
            ids = np.array([3, 1, 0], np.int32)
            got = be.sample(ids, 5, None, 0.5, seed=99, call=step, attempts=200)
            want = port.sample(ids, 5, replay_uniforms(99, step, 15, 200), 0.5)
            for name in ("tree_idx", "states", "actions", "next_states", "nonterminals", "returns", "attempts", "error"):
                np.testing.assert_array_equal(got[name], want[name], err_msg=name)
            assert rc.ulp_diff(got["weights"], want["weights"]).max() <= 1
            for e in want["error"][want["error"] != 0]:
                expect |= 1 << int(e)
            ok = got["tree_idx"] >= 0
            rows_m = np.repeat(ids, 5)[ok]
            rows_i = got["tree_idx"][ok]
            loss = (rng.random(ok.sum()) * 2).astype(np.float32)
            rows_m, rows_i, loss = np.append(rows_m, rows_m[0]), np.append(rows_i, rows_i[0]), np.append(loss, 0.25)
            be.update(rows_m, rows_i, loss); port.update_priorities(rows_m, rows_i, loss)
            tree, *_blk = be.snapshot()
            # numpy's float32 power is not always correctly rounded for omega = 0.6: leaves within 1 ulp
            assert rc.ulp_diff(tree[:, C - 1:], port.tree[:, C - 1:]).max() <= 1
            be.a["tree"][:] = port.tree                       # continue from identical trees
            be.a["state"][:, 3] = port.max.view(np.int32)
    assert be.flags[0] == expect
    be.flags[0] = 0
    be.update(np.array([0, 7], np.int32), np.array([C - 1, C - 1], np.int64), np.ones(2, np.float32))
    be.update(np.array([0], np.int32), np.array([2 * C - 1], np.int64), np.ones(1, np.float32))
    assert be.flags[0] == 1 << 3


def test_emulated_kernels_bound_starved_stratum(emu_lib):
    be = EmuBackend(emu_lib, 1, 16, 5, n=3)
    for k in range(12):
        be.append(np.full((1, 5), float(k), np.float32), [k % 4], [0.5 * k], [k % 5 == 4], [1], 0.0)
    want = starved_port().sample([0], 4, replay_uniforms(7, 0, 4, 64))
    got = be.sample(np.zeros(1, np.int32), 4, None, 0.4, seed=7, call=0, attempts=64)
    assert list(got["error"]) == [0, 0, 0, ERR_STARVED]
    for name in ("tree_idx", "attempts", "error", "states", "returns"):
        np.testing.assert_array_equal(got[name], want[name], err_msg=name)
    assert be.flags[0] == 1 << ERR_STARVED
    got = be.sample(np.array([0, 5], np.int32), 1, None, 0.4, attempts=8)
    assert list(got["error"]) == [0, 2]


def test_replay_calls_validate_arguments():
    """Argument validation happens before any CUDA call, so the product library is checkable here."""
    from irbpp_b200 import _lib, build
    build.build()
    lib = _lib.load()
    dummy = np.zeros(64, np.float32)
    p = ptr(dummy)
    mem = _lib.IrbppReplayMemory(4, 1, 8, p, p, p, p, p, p, p)            # C = 1
    assert lib.irbpp_replay_init(ctypes.byref(mem), None) == _lib.IRBPP_EINVAL
    assert b"C >= 2" in lib.irbpp_last_error(None)
    mem.capacity = 8
    batch = _lib.IrbppReplayBatch(p, p, p, p, p, p, p, None, None)
    call = lambda G, k, n, A: lib.irbpp_replay_sample(ctypes.byref(mem), p, G, k, n, 0.99, 0.4, A, 0, 0, None,
                                                      ctypes.byref(batch), None, None)
    assert call(1, 0, 3, 10) == _lib.IRBPP_EINVAL            # k >= 1
    assert call(0, 1, 3, 10) == _lib.IRBPP_EINVAL
    assert call(1, 1, 8, 10) == _lib.IRBPP_EINVAL            # n < C
    assert call(1, 1, 3, 0) == _lib.IRBPP_EINVAL             # attempts >= 1
    assert lib.irbpp_replay_update_priorities(ctypes.byref(mem), p, p, p, 0, 0.5, None, None) == _lib.IRBPP_EINVAL
    assert lib.irbpp_replay_append(ctypes.byref(mem), p, 4, p, p, p, None, 0.0, None) == _lib.IRBPP_EINVAL   # stride
    mem.tree = None
    assert lib.irbpp_replay_init(ctypes.byref(mem), None) == _lib.IRBPP_EINVAL
