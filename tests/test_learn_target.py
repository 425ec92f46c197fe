"""The target half of ``Agent.learn`` without a GPU: ``irbpp_dqn_target`` / ``irbpp_dqn_order_target`` under the host
emulator against the float64 port (``oracle/learn_port.py``), their projection against a NumPy float32 restatement
of the kernel's order of operations, the edge cases of ``agent.py:100-115`` and the argument checks.

Bars: ``|p - p64| <= 3e-6`` per atom (``p64`` the float64 port's ``p(s', a*)`` from the same effective weights and
the kernel's a*); per transition ``|sum m - sum p| <= 1e-6`` and ``sum |m - m64| <= sum |p - p64| + 2 max |b - b64|
+ 1e-6``.  The middle term is the float32 evaluation of ``b = (Tz - Vmin) / dz`` that torch's float32 expression
(and so the kernel) carries: an error d in b moves 2 p d of mass between l and u.  On the reference's support
(dz = 0.3) it reaches a few 1e-6; on an exact grid (dz = 1) it is 0 and the bar is ``sum |p - p64| + 1e-6``."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.learn_port import project64, target64
from test_actor_range import make_bins, seeded_net, shape_features
from test_order_actor import make_obs, seeded_net as seeded_order_net, shape_table

pytestmark = pytest.mark.timeout(900)

P_TOL = 3e-6
M_TOL = 1e-6
DEFAULT = dict(v_min=-1.0, v_max=8.0, discount_n=0.99 ** 3)       # the reference's V_min, V_max, discount ** multi_step
SELS = (1, 7, 500)
KS = (2, 10, 32)
ATOMS = (2, 31, 32)


@pytest.fixture(scope="module")
def fx():
    from test_actor import decode_fixture
    from conftest import load_golden
    return decode_fixture(load_golden("dqn_act"))


@pytest.fixture(scope="module")
def order_fx():
    from test_order_actor import decode_fixture
    from conftest import load_golden
    return decode_fixture(load_golden("dqn_order_act"))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    from irbpp_b200._lib import SIGNATURES
    from test_kernels_emulated import build_emulated
    lib = build_emulated(str(tmp_path_factory.mktemp("emu_learn")))
    for name in ("irbpp_dqn_target", "irbpp_dqn_scratch_bytes", "irbpp_dqn_order_target", "irbpp_dqn_order_scratch_bytes"):
        fn = getattr(lib, "emu_" + name)
        fn.restype, fn.argtypes = SIGNATURES[name]
    return lib


# ---- the call ----

def _addr(a):
    return a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data


def effective(net32, fields):
    from irbpp_b200.actor import NOISY
    sd = net32.state_dict()
    eff = {k: sd[k] for _, k in fields if k in sd}
    with torch.no_grad():
        for m in NOISY:
            eff[m + ".weight"], eff[m + ".bias"] = getattr(net32, m).effective()
    return eff


def dqn_target(lib, level, net32, obs, size, sf, support, next_actions, returns, nonterminals, v_min, v_max,
               discount_n, prefix="emu_", want_p=True):
    """``irbpp_dqn_target`` (level ``"location"``, ``size`` = selected_action) or ``irbpp_dqn_order_target``
    (``"order"``, ``size`` = k; ``sf`` the per-shape table) with the port's effective weights.  NumPy arrays for the
    emulated library, CUDA tensors for the real one (``prefix=""``).  Returns ``(rc, m, p)`` as NumPy."""
    from irbpp_b200._lib import IrbppDqnOrderWeights, IrbppDqnWeights
    from irbpp_b200.actor import _FIELDS, _ORDER_FIELDS
    fields, W = (_FIELDS, IrbppDqnWeights) if level == "location" else (_ORDER_FIELDS, IrbppDqnOrderWeights)
    dev = obs.device if isinstance(obs, torch.Tensor) else None
    eff = effective(net32, fields)
    B, atoms = obs.shape[0], len(support)
    if dev is None:
        keep = {f: np.ascontiguousarray(eff[k].detach().cpu().numpy(), np.float32) for f, k in fields}
        arr = lambda a, t: np.ascontiguousarray(a, t)
        sf, support = arr(sf, np.float32), arr(support, np.float32)
        a, r, nt = arr(next_actions, np.int64), arr(returns, np.float32), arr(nonterminals, np.float32)
        m, p = np.full((B, atoms), np.nan, np.float32), np.full((B, atoms), np.nan, np.float32)
        stream = None
    else:
        keep = {f: eff[k].detach().to(dev, torch.float32).contiguous() for f, k in fields}
        arr = lambda a, t: torch.as_tensor(a).to(dev, t).contiguous()
        sf, support = arr(sf, torch.float32), arr(support, torch.float32)
        a, r, nt = arr(next_actions, torch.int64), arr(returns, torch.float32), arr(nonterminals, torch.float32)
        m = torch.full((B, atoms), float("nan"), device=dev)
        p = torch.full((B, atoms), float("nan"), device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
    w = W(*([_addr(keep[f]) for f, _ in fields] + [ctypes.c_float(0.01)]))
    row = obs.stride(0) if dev is not None else obs.strides[0] // 4
    if level == "location":
        nbytes = getattr(lib, prefix + "irbpp_dqn_scratch_bytes")(B, size)
    else:
        nbytes = getattr(lib, prefix + "irbpp_dqn_order_scratch_bytes")(B, size, sf.shape[0])
    if dev is None:
        raw = np.zeros(nbytes + 256, np.uint8)
        scratch = raw.ctypes.data + (-raw.ctypes.data) % 256
    else:
        raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        scratch = raw.data_ptr() + (-raw.data_ptr()) % 256
    tail = (_addr(a), _addr(r), _addr(nt), discount_n, v_min, v_max, _addr(m), _addr(p) if want_p else None, scratch,
            nbytes, stream)
    if level == "location":
        rc = getattr(lib, prefix + "irbpp_dqn_target")(ctypes.byref(w), _addr(obs), row, B, size, _addr(sf),
                                                       _addr(support), atoms, *tail)
    else:
        rc = getattr(lib, prefix + "irbpp_dqn_order_target")(ctypes.byref(w), _addr(obs), row, B, size, _addr(sf),
                                                             sf.shape[0], _addr(support), atoms, *tail)
    if dev is not None:
        torch.cuda.synchronize(dev)
        m, p = m.cpu(), p.cpu()
    return rc, np.asarray(m), np.asarray(p)


def project32(p, returns, nonterminals, support, v_min, v_max, discount_n):
    """The kernel's projection (csrc/irbpp_learn.cuh) restated in NumPy float32: one rounding per operation, the
    division as a multiplication by the float32 reciprocal of dz, l-contributions in atom order, then
    u-contributions in atom order, each added to m in that order; b capped at atoms - 1, where torch's float32 b can
    pass it by an ulp (csrc/irbpp_learn.cuh)."""
    f = np.float32
    p = np.asarray(p, f)
    B, atoms = p.shape
    z = np.asarray(support, f)[None, :]
    R = np.asarray(returns, f).reshape(B, 1)
    nt = np.asarray(nonterminals, f).reshape(B, 1)
    vmin, vmax = f(v_min), f(v_max)
    inv = f(1.0) / f((v_max - v_min) / (atoms - 1))
    tz = R + (nt * f(discount_n)) * z
    tz = np.minimum(np.maximum(tz, vmin), vmax)
    b = np.minimum((tz - vmin) * inv, f(atoms - 1))
    l, u = np.floor(b).astype(np.int64), np.ceil(b).astype(np.int64)
    l[(u > 0) & (l == u)] -= 1
    u[(l < atoms - 1) & (l == u)] += 1
    cl, cu = p * (u.astype(f) - b), p * (b - l.astype(f))
    m = np.zeros((B, atoms), f)
    for r in range(B):
        for i in range(atoms):
            m[r, l[r, i]] += cl[r, i]
        for i in range(atoms):
            m[r, u[r, i]] += cu[r, i]
    return m, b


def check_bars(m, p, ref, b32):
    """The accuracy bars against ``target64``'s output (``b32``: the float32 b); returns (worst |p - p64|, worst l1
    excess of m over sum |p - p64|)."""
    dp = np.abs(p - ref["p"])
    assert dp.max() <= P_TOL, dp.max()
    l1m = np.abs(m - ref["m"]).sum(1)
    db = np.abs(b32.astype(np.float64) - ref["b"]).max(1)
    assert (l1m <= dp.sum(1) + 2 * db + M_TOL).all(), (l1m - dp.sum(1) - 2 * db).max()
    assert (np.abs(m.astype(np.float64).sum(1) - p.astype(np.float64).sum(1)) <= M_TOL).all()
    return float(dp.max()), float((l1m - dp.sum(1)).max())


# ---- the inputs ----

def transitions(B, size, seed, v_min, v_max):
    """a* over the rows (every row, valid or not), returns reaching past both ends of the support, nonterminals
    0 and 1."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, size, B).astype(np.int64)
    span = v_max - v_min
    R = rng.uniform(v_min - 0.3 * span, v_max + 0.3 * span, B).astype(np.float32)
    nt = (rng.random(B) < 0.7).astype(np.float32)
    nt[0] = 0.0
    return a, R, nt


def location_case(fx, sel, atoms, mode, seed=0):
    net = seeded_net(sel, atoms, mode)
    n_valid = [min(sel, v) for v in (0, 1, sel // 2, sel)]
    obs, src = make_bins(fx, sel, n_valid, seed=sel + atoms)
    obs[0] = 0.0                                                # a blank next state (memory.py:106): no valid row
    sf = shape_features(fx, net, src).numpy()
    return net, obs, sf


def order_case(ofx, k, atoms, mode):
    net = seeded_order_net(k, atoms, mode)
    B = 64 // k + 1                                             # two tiles of the slots kernel, the second partial
    obs = make_obs(ofx, k, B, ofx["clouds"].shape[0], seed=k * 7 + atoms)
    obs[0] = 0.0                                                # a blank next state
    sf = shape_table(net, ofx["clouds"]).numpy()
    return net, obs, sf


def run(emu, level, net, obs, size, sf, atoms, a, R, nt, v_min, v_max, discount_n):
    support = np.linspace(v_min, v_max, atoms).astype(np.float32)      # torch.linspace's float32 support
    rc, m, p = dqn_target(emu, level, net, obs, size, sf, support, a, R, nt, v_min, v_max, discount_n)
    assert rc == 0, rc
    ref = target64(None, net, obs, None, sf, support, R, nt, v_min, v_max, discount_n,
                   next_actions=np.clip(a, 0, size - 1))                   # the entry points clamp a*
    return m, p, ref, support


# ---- the tests ----

@pytest.mark.parametrize("atoms", ATOMS)
@pytest.mark.parametrize("sel", SELS)
def test_emulated_location_target(fx, emu, sel, atoms):
    for mode in ("train", "eval"):
        net, obs, sf = location_case(fx, sel, atoms, mode)
        a, R, nt = transitions(obs.shape[0], sel, sel * 3 + atoms, DEFAULT["v_min"], DEFAULT["v_max"])
        m, p, ref, support = run(emu, "location", net, obs, sel, sf, atoms, a, R, nt, **DEFAULT)
        m32, b32 = project32(p, R, nt, support, **DEFAULT)
        worst = check_bars(m, p, ref, b32)
        assert np.array_equal(m, m32)
        print("location sel %d atoms %d %s: |p - p64| %.3g, m excess %.3g" % ((sel, atoms, mode) + worst))


@pytest.mark.parametrize("atoms", ATOMS)
@pytest.mark.parametrize("k", KS)
def test_emulated_order_target(order_fx, emu, k, atoms):
    for mode in ("train", "eval"):
        net, obs, sf = order_case(order_fx, k, atoms, mode)
        a, R, nt = transitions(obs.shape[0], k, k * 3 + atoms, DEFAULT["v_min"], DEFAULT["v_max"])
        m, p, ref, support = run(emu, "order", net, obs, k, sf, atoms, a, R, nt, **DEFAULT)
        m32, b32 = project32(p, R, nt, support, **DEFAULT)
        worst = check_bars(m, p, ref, b32)
        assert np.array_equal(m, m32)
        print("order k %d atoms %d %s: |p - p64| %.3g, m excess %.3g" % ((k, atoms, mode) + worst))


def test_projection_is_bit_exact_against_numpy_float32(fx, emu):
    """The kernel's m equals the NumPy float32 restatement bit for bit, given the kernel's own p: both round each
    operation once in the same order and add the contributions in the same order, so there is nothing to tolerate.
    Many transitions on one bin, the reference's support and an uneven discount."""
    net, obs, sf = location_case(fx, 7, 31, "train")
    B = 64
    obs, sf = np.repeat(obs[2:3], B, 0), np.repeat(sf[2:3], B, 0)
    a, R, nt = transitions(B, 7, 11, -1.0, 8.0)
    kw = dict(v_min=-1.0, v_max=8.0, discount_n=0.97 ** 5)
    m, p, ref, support = run(emu, "location", net, obs, 7, sf, 31, a, R, nt, **kw)
    m32, b32 = project32(p, R, nt, support, **kw)
    assert np.array_equal(m, m32)
    worst = check_bars(m, p, ref, b32)
    print("64 transitions: |p - p64| %.3g, m excess %.3g, max |b - b64| %.3g" % (worst + (np.abs(b32 - ref["b"]).max(),)))


def test_edge_cases_on_an_exact_grid(fx, emu):
    """Support -10..10 with 21 atoms (dz = 1, every b exact in float32 and float64): b an integer in the interior, at
    0 and at atoms - 1 (l == u, both fix-ups), Tz clamped at both ends, terminal transitions, and a blank next state
    with zero valid rows."""
    kw = dict(v_min=-10.0, v_max=10.0, discount_n=1.0)
    R = np.array([3.0, -10.0, 10.0, -25.0, 25.0, 0.0, 2.5, -4.0], np.float32)
    nt = np.array([0, 0, 0, 1, 1, 1, 0, 1], np.float32)
    B = len(R)
    net, obs, sf = location_case(fx, 7, 21, "train")
    obs, sf = obs[np.arange(B) % 4], sf[np.arange(B) % 4]
    obs[1] = 0.0
    a = np.arange(B, dtype=np.int64) % 7
    m, p, ref, support = run(emu, "location", net, obs, 7, sf, 21, a, R, nt, **kw)
    m32, b32 = project32(p, R, nt, support, **kw)
    assert np.array_equal(b32, ref["b"])                            # dz = 1: b exact in float32
    check_bars(m, p, ref, b32)
    assert np.array_equal(m, m32)
    exact = project64(p, R, nt, support, **kw)["m"]                 # same l and u: m64 of the kernel's own p
    np.testing.assert_allclose(m, exact, rtol=0, atol=1e-7)
    one = lambda r, j: np.eye(21)[j] * p[r].astype(np.float64).sum()
    np.testing.assert_allclose(m[0], one(0, 13), atol=1e-6)         # b = 13: all mass on atom 13 (l = 12 gets 0)
    np.testing.assert_allclose(m[1], one(1, 0), atol=1e-6)          # b = 0: l == u == 0, u moves to 1 with weight 0
    np.testing.assert_allclose(m[2], one(2, 20), atol=1e-6)         # b = 20 = atoms - 1: l moves to 19
    assert (m[0] != 0).sum() == 1 and (m[1] != 0).sum() == 1 and (m[2] != 0).sum() == 1
    np.testing.assert_allclose(m[3], one(3, 0), atol=1e-6)          # Tz = -25 + z <= -10 everywhere
    np.testing.assert_allclose(m[4], one(4, 20), atol=1e-6)         # Tz = 25 + z >= 10 everywhere
    np.testing.assert_allclose(m[5], p[5], atol=0)                  # Tz = z: every b an integer, m = p
    np.testing.assert_allclose(m[6], (one(6, 12) + one(6, 13)) / 2, atol=1e-6)   # b = 12.5: half to each side


def test_out_of_range_actions_are_clamped(fx, order_fx, emu):
    net, obs, sf = location_case(fx, 7, 31, "eval")
    B = obs.shape[0]
    R, nt = np.full(B, 1.5, np.float32), np.ones(B, np.float32)
    kw = dict(v_min=-1.0, v_max=8.0, discount_n=0.9)
    wild = np.array([-5, 7, 1 << 40, -(1 << 40)], np.int64)
    m1, p1, _, _ = run(emu, "location", net, obs, 7, sf, 31, wild, R, nt, **kw)
    m2, p2, _, _ = run(emu, "location", net, obs, 7, sf, 31, np.clip(wild, 0, 6), R, nt, **kw)
    assert np.array_equal(m1, m2) and np.array_equal(p1, p2)
    onet, oobs, osf = order_case(order_fx, 10, 31, "train")
    B = oobs.shape[0]
    wild = np.resize(np.array([-1, 10, 99, 3], np.int64), B)
    R, nt = np.linspace(-2, 9, B).astype(np.float32), np.ones(B, np.float32)
    m1, p1, _, _ = run(emu, "order", onet, oobs, 10, osf, 31, wild, R, nt, **kw)
    m2, p2, _, _ = run(emu, "order", onet, oobs, 10, osf, 31, np.clip(wild, 0, 9), R, nt, **kw)
    assert np.array_equal(m1, m2) and np.array_equal(p1, p2)


def test_b_is_capped_at_the_last_atom(fx, emu):
    """32 atoms on [-1, 8]: at Tz = Vmax the float32 b is 9 * float32(31 / 9) = 31.000002, past the last atom (torch's
    index_add_ would add into the next transition's row there).  The kernel caps b at atoms - 1: all of p stays in the
    transition's own m and m equals the float64 projection's."""
    kw = dict(v_min=-1.0, v_max=8.0, discount_n=1.0)
    f = np.float32
    assert (f(8.0) - f(-1.0)) * (f(1.0) / f(9.0 / 31)) > f(31)
    net, obs, sf = location_case(fx, 7, 32, "train")
    B = obs.shape[0]
    R, nt = np.array([8.0, 20.0, 8.0, -1.0], np.float32)[:B], np.zeros(B, np.float32)
    a = np.arange(B, dtype=np.int64)
    m, p, ref, support = run(emu, "location", net, obs, 7, sf, 32, a, R, nt, **kw)
    assert np.array_equal(m, project32(p, R, nt, support, **kw)[0])
    np.testing.assert_allclose(m.astype(np.float64).sum(1), p.astype(np.float64).sum(1), rtol=0, atol=1e-6)
    np.testing.assert_allclose(m, ref["m"], rtol=0, atol=1e-6)


def test_argument_checks(emu):
    """atoms 1 and 33, v_max <= v_min, B < 1 and a NULL m are refused with IRBPP_EINVAL; p_next may be NULL."""
    from irbpp_b200._lib import IRBPP_EINVAL, IrbppDqnOrderWeights, IrbppDqnWeights
    buf = np.zeros(1 << 16, np.float32)
    a = np.zeros(4, np.int64)
    nbytes = emu.emu_irbpp_dqn_scratch_bytes(4, 7)
    raw = np.zeros(nbytes + 256, np.uint8)
    scratch = raw.ctypes.data + (-raw.ctypes.data) % 256
    w = IrbppDqnWeights(*([buf.ctypes.data] * 22 + [ctypes.c_float(0.01)]))

    def call(atoms=31, vmin=-1.0, vmax=8.0, B=4, m=buf.ctypes.data):
        return emu.emu_irbpp_dqn_target(ctypes.byref(w), buf.ctypes.data, 7 * 5 + 9 + 1024, B, 7, buf.ctypes.data,
                                        buf.ctypes.data, atoms, a.ctypes.data, buf.ctypes.data, buf.ctypes.data, 0.9,
                                        vmin, vmax, m, None, scratch, nbytes, None)
    for kw in (dict(atoms=1), dict(atoms=33), dict(vmin=8.0), dict(vmin=9.0), dict(B=0), dict(m=None)):
        assert call(**kw) == IRBPP_EINVAL, kw
    onb = emu.emu_irbpp_dqn_order_scratch_bytes(4, 10, 8)
    oraw = np.zeros(onb + 256, np.uint8)
    oscratch = oraw.ctypes.data + (-oraw.ctypes.data) % 256
    ow = IrbppDqnOrderWeights(*([buf.ctypes.data] * 27 + [ctypes.c_float(0.01)]))

    def ocall(atoms=31, vmin=-1.0, vmax=8.0, B=4, k=10):
        return emu.emu_irbpp_dqn_order_target(ctypes.byref(ow), buf.ctypes.data, 1034, B, k, buf.ctypes.data, 8,
                                              buf.ctypes.data, atoms, a.ctypes.data, buf.ctypes.data, buf.ctypes.data,
                                              0.9, vmin, vmax, buf.ctypes.data, None, oscratch, onb, None)
    for kw in (dict(atoms=1), dict(atoms=33), dict(vmax=-1.0), dict(B=0), dict(k=1), dict(k=33)):
        assert ocall(**kw) == IRBPP_EINVAL, kw
