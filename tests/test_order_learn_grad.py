"""The gradient pass of ``Agent.learn`` at the order level without a GPU: ``irbpp_dqn_order_log_prob`` and
``irbpp_dqn_order_log_prob_backward`` under the host emulator against the float64 port (``OrderDQNPort`` through
``oracle.learn_port.distribution(..., log=True)`` with ``torch.autograd``).

Bars (``tests/test_learn_grad.py``'s): forward ``|log p - log p64| <= EMU_RTOL (1 + |log p64|)``; backward, for each of
the 21 tensors and both feature gradients, ``max |grad - grad64| <= 1e-4 max |grad64|``, or twice torch float32's own
error on the same inputs where that is larger.  The port runs in float64 from the same effective weights: NoisyLinear
layers in train mode become eval-mode layers whose ``mu`` is the effective tensor, the height encoder a constant
``map_feature`` leaf, and the per-shape features ``[S, 128]`` a leaf the slots gather from."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from oracle.learn_port import distribution
from test_learn_grad import EMU_RTOL, GRAD_RTOL, _Const, check_grads, dq_scale, forward_error
from test_order_actor import decode_fixture, make_obs, port_from, seeded_net, shape_table

pytestmark = pytest.mark.timeout(1800)

KS = (2, 10, 32)
ATOMS = (1, 2, 31, 32)
HM = 32


@pytest.fixture(scope="module")
def fx():
    from conftest import load_golden
    return decode_fixture(load_golden("dqn_order_act"))


def emulated_library(tmp):
    from irbpp_b200._lib import SIGNATURES
    from test_kernels_emulated import build_emulated
    lib = build_emulated(tmp)
    for name in ("irbpp_dqn_order_log_prob", "irbpp_dqn_order_log_prob_backward",
                 "irbpp_dqn_order_log_prob_scratch_bytes"):
        fn = getattr(lib, "emu_" + name)
        fn.restype, fn.argtypes = SIGNATURES[name]
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emulated_library(str(tmp_path_factory.mktemp("emu_order_learn_grad")))


# ---- the calls ----

def _addr(a):
    return a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data


def order_tensors(net32):
    """The effective tensors of ``net32`` after the convolutions, by field of ``irbpp_dqn_order_grads`` (float32)."""
    from irbpp_b200.actor import NOISY, _ORDER_ROW_FIELDS
    sd = net32.state_dict()
    eff = {}
    with torch.no_grad():
        for m in NOISY:
            eff[m + ".weight"], eff[m + ".bias"] = getattr(net32, m).effective()
    return {f: (eff[k] if k in eff else sd[k]).detach().float() for f, k in _ORDER_ROW_FIELDS}


def order_log_prob_calls(lib, net32, obs, k, sf, mf, actions, g=None, prefix="emu_"):
    """``irbpp_dqn_order_log_prob`` and, when ``g`` is given, ``irbpp_dqn_order_log_prob_backward`` with the port's
    effective weights.  NumPy inputs for the emulated library, CUDA tensors for the real one (``prefix=""``).  Returns
    ``(rc, log_p, grads)`` with ``grads`` a dict field -> array plus ``"shape_features"`` / ``"map_feature"`` (None
    without ``g``), all NumPy."""
    from irbpp_b200._lib import IrbppDqnOrderGrads, IrbppDqnOrderWeights
    from irbpp_b200.actor import _ORDER_FIELDS, _ORDER_ROW_FIELDS
    dev = obs.device if isinstance(obs, torch.Tensor) else None
    ws = order_tensors(net32)
    B, atoms, S = obs.shape[0], ws["fc_z_a_b"].shape[0], sf.shape[0]
    if dev is None:
        conv = lambda a, t: np.ascontiguousarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a, t)
        new = lambda shape: np.full(shape, np.nan, np.float32)
        row = obs.strides[0] // 4
    else:
        conv = lambda a, t: torch.as_tensor(a).to(dev, {np.float32: torch.float32, np.int64: torch.int64}[t]).contiguous()
        new = lambda shape: torch.full(shape, float("nan"), device=dev)
        row = obs.stride(0)
    keep = {f: conv(ws[f], np.float32) for f, _ in _ORDER_ROW_FIELDS}
    sf, mf, a = conv(sf, np.float32), conv(mf, np.float32), conv(actions, np.int64)
    w = IrbppDqnOrderWeights(*([_addr(keep[f]) if f in keep else None for f, _ in _ORDER_FIELDS] + [ctypes.c_float(0.01)]))
    nbytes = getattr(lib, prefix + "irbpp_dqn_order_log_prob_scratch_bytes")(B, k, S)
    if dev is None:
        raw = np.zeros(nbytes + 256, np.uint8)
        scratch, stream = raw.ctypes.data + (-raw.ctypes.data) % 256, None
    else:
        raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        scratch, stream = raw.data_ptr() + (-raw.data_ptr()) % 256, torch.cuda.current_stream(dev).cuda_stream
    log_p = new((B, atoms))
    rc = getattr(lib, prefix + "irbpp_dqn_order_log_prob")(ctypes.byref(w), _addr(obs), row, B, k, _addr(sf), S,
                                                           _addr(mf), _addr(a), atoms, _addr(log_p), scratch, nbytes,
                                                           stream)
    grads = None
    if rc == 0 and g is not None:
        gg = conv(g, np.float32)
        out = {f: new(tuple(keep[f].shape)) for f, _ in _ORDER_ROW_FIELDS}
        out["shape_features"], out["map_feature"] = new((S, 128)), new((B, 256))
        d = IrbppDqnOrderGrads(*[_addr(out[f]) for f, _ in _ORDER_ROW_FIELDS])
        rc = getattr(lib, prefix + "irbpp_dqn_order_log_prob_backward")(
            ctypes.byref(w), _addr(obs), row, B, k, _addr(sf), S, _addr(mf), _addr(a), atoms, _addr(gg), ctypes.byref(d),
            _addr(out["shape_features"]), _addr(out["map_feature"]), scratch, nbytes, stream)
        grads = out
    if dev is not None:
        torch.cuda.synchronize(dev)
        log_p = log_p.cpu()
        grads = None if grads is None else {key: v.cpu() for key, v in grads.items()}
    to_np = lambda x: x.numpy() if isinstance(x, torch.Tensor) else x
    return rc, to_np(log_p), None if grads is None else {key: to_np(v) for key, v in grads.items()}


def order_port_grads(net32, obs, sf, mf, actions, g, dtype=torch.float64):
    """``log p(s, a_t, .)`` and the gradients of ``sum(g * log p)`` with respect to the effective tensors, the
    per-shape features and the map features, by ``torch.autograd`` on the port in ``dtype``, on the device the inputs
    live on."""
    from irbpp_b200.actor import NOISY, _ORDER_ROW_FIELDS
    t = lambda a: (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))).to(dtype)
    obs = t(obs)
    dev = obs.device
    eff = order_tensors(net32)
    net = copy.deepcopy(net32).to(dev, dtype)
    with torch.no_grad():
        for m in NOISY:
            getattr(net, m).weight_mu.copy_(eff["%s_w" % m])
            getattr(net, m).bias_mu.copy_(eff["%s_b" % m])
    net.eval()
    sf_leaf = t(sf).to(dev).requires_grad_(True)
    mf_leaf = t(mf).to(dev).requires_grad_(True)
    net.heightEncoder = _Const(mf_leaf)
    B, k = obs.shape[0], net.k
    a = torch.as_tensor(np.clip(np.asarray(actions), 0, k - 1), device=dev)
    lp = distribution(net, obs, sf_leaf, log=True)[torch.arange(B, device=dev), a]
    (lp * t(g).to(dev)).sum().backward()
    params = dict(net.named_parameters())
    out = {}
    for f, key in _ORDER_ROW_FIELDS:
        name = key.replace(".weight", ".weight_mu").replace(".bias", ".bias_mu") if key.split(".")[0] in NOISY else key
        grad = params[name].grad
        out[f] = np.zeros(tuple(params[name].shape)) if grad is None else grad.detach().cpu().double().numpy()
    out["shape_features"] = sf_leaf.grad.detach().cpu().double().numpy()
    out["map_feature"] = mf_leaf.grad.detach().cpu().double().numpy()
    return lp.detach().cpu().double().numpy(), out


# ---- the inputs ----

def map_features(net32, obs, k):
    """The height encoder of ``net32`` on the order observations' heightmaps (float32)."""
    B = obs.shape[0]
    hm = torch.from_numpy(np.ascontiguousarray(obs[:, k:k + HM * HM])).reshape(B, 1, HM, HM)
    with torch.no_grad():
        return net32.heightEncoder(hm).reshape(B, -1).numpy()


def shape_rows(fx, net32, S, seed):
    """S per-shape features around the fixture shapes' features through ``net32``'s encoder.  The fixture's clouds
    give nearly equal features (their spread is ~3e-4 of a value), which makes every slot of a bin alike: the
    attention's gradient then cancels to rounding in float32 and float64 alike.  Seeded rows with the features' own
    spread (0.075) keep the slots apart."""
    base = shape_table(net32, fx["clouds"]).numpy()
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(base.mean(0) + base.std() * rng.normal(size=(S, 128)), np.float32)


def order_case(fx, net, k, B, S, seed=0):
    """B order observations (the fixture's heightmaps) whose ids repeat within and across bins and include some
    outside [0, S) (clamped); a_t random, two of them out of range (clamped); g random."""
    rng = np.random.default_rng(seed + 31 * k + B)
    obs = make_obs(fx, k, B, S, seed=seed + k)
    ids = rng.integers(-2, S + 3, (B, k)).astype(np.float32)
    ids[:, 1] = ids[:, 0]                                        # a duplicate within every bin
    if B > 1:
        ids[1, 2 % k] = ids[0, 0]                                # and across bins
    obs[:, :k] = ids
    sf = shape_rows(fx, net, S, seed)
    mf = map_features(net, obs, k)
    actions = rng.integers(0, k, B).astype(np.int64)
    actions[0] = -1
    actions[-1] = k + 2 if B > 1 else actions[-1]
    g = rng.normal(size=(B, net.atoms)).astype(np.float32)
    return obs, sf, mf, actions, g


# with every slot of a bin alike: gradient -> the gradient of the same size that does not cancel
ALIKE_SCALE = {"wq": "wv", "wk": "wv", "fc_h_a_w": "fc_h_v_w", "fc_h_a_b": "fc_h_v_b", "fc_z_a_w": "fc_z_v_w"}


def check_order_grads(grads, ref, label, bias_scale, ref32, alike=False):
    """``check_grads``; with ``alike`` (every slot of a bin holds the same shape, so the slots are equal) the gradients
    of W_query and W_key (the softmax's gradient sums to zero over equal slots) and of the advantage stream's weights
    (``sum_j da_j = 0`` times equal activations) are zero in real arithmetic, and what float32 returns is rounding of
    terms that cancel: each is held to GRAD_RTOL of the gradient in ``ALIKE_SCALE``, the size of those terms."""
    if alike:
        for key, other in ALIKE_SCALE.items():
            err = np.abs(np.asarray(grads[key], np.float64) - ref[key]).max() / np.abs(ref[other]).max()
            print("%s %-14s kernel %.3g of max |d %s|" % (label, key, err, other))
            assert err <= GRAD_RTOL, (label, key, err)
        grads, ref, ref32 = ({key: v for key, v in d.items() if key not in ALIKE_SCALE} for d in (grads, ref, ref32))
    return check_grads(grads, ref, label, bias_scale, ref32)


def check_case(lib, net, obs, k, sf, mf, a, g, label):
    rc, lp, grads = order_log_prob_calls(lib, net, obs, k, sf, mf, a, g)
    assert rc == 0, rc
    lp64, ref = order_port_grads(net, obs, sf, mf, a, g)
    lp32, ref32 = order_port_grads(net, obs, sf, mf, a, g, dtype=torch.float32)
    err = forward_error(lp, lp64)
    print("%s: |log p - log p64| / (1 + |log p64|) %.3g (torch float32 %.3g)" % (label, err, forward_error(lp32, lp64)))
    assert np.isfinite(lp).all() and err <= EMU_RTOL, err
    return check_order_grads(grads, ref, label, dq_scale(lp64, g), ref32, alike=sf.shape[0] == 1)


# ---- the tests ----

@pytest.mark.parametrize("atoms", ATOMS)
@pytest.mark.parametrize("k", KS)
def test_emulated_log_prob_and_backward(fx, emu, k, atoms):
    """7 bins over a library of 5 shapes (ids repeat and run out of range).  The mode alternates over the grid, so
    every k and every atom count runs in train and in eval mode; at 31 atoms the weights are the reference fixture's,
    elsewhere seeded with the reference's initialisation rules."""
    mode = ("train", "eval")[(KS.index(k) + ATOMS.index(atoms)) % 2]
    net = port_from(fx, k, mode == "train", torch.float32) if atoms == 31 else seeded_net(k, atoms, mode)
    obs, sf, mf, a, g = order_case(fx, net, k, 7, 5)
    label = "k %d atoms %d %s%s" % (k, atoms, mode, " fixture" if atoms == 31 else "")
    check_case(emu, net, obs, k, sf, mf, a, g, label)


@pytest.mark.parametrize("B,S", [(1, 1), (64, 700)])
def test_emulated_batch_and_library_sizes(fx, emu, B, S):
    """B = 1 and B = 64 at k = 10: a library of one shape (every id clamps to it, every slot of the bin is alike) and
    one of more shapes than slots (most get no gradient)."""
    net = seeded_net(10, 31, "train")
    obs, sf, mf, a, g = order_case(fx, net, 10, B, S, seed=2)
    check_case(emu, net, obs, 10, sf, mf, a, g, "B %d S %d" % (B, S))


def test_two_runs_are_bit_identical(fx, emu):
    net = seeded_net(10, 31, "train")
    obs, sf, mf, a, g = order_case(fx, net, 10, 9, 4, seed=3)
    r1 = order_log_prob_calls(emu, net, obs, 10, sf, mf, a, g)
    r2 = order_log_prob_calls(emu, net, obs, 10, sf, mf, a, g)
    assert np.array_equal(r1[1], r2[1])
    for key in r1[2]:
        assert np.array_equal(r1[2][key], r2[2][key]), key


def test_argument_checks(emu):
    """B < 1, k outside [2, 32], atoms outside [1, 32], S < 1, NULL inputs, weights and outputs, a short observation
    stride, a short or misaligned scratch are refused with IRBPP_EINVAL."""
    from irbpp_b200._lib import IRBPP_EINVAL, IrbppDqnOrderGrads, IrbppDqnOrderWeights
    buf = np.zeros(1 << 16, np.float32)
    a = np.zeros(4, np.int64)
    p = buf.ctypes.data
    nbytes = emu.emu_irbpp_dqn_order_log_prob_scratch_bytes(4, 10, 8)
    assert nbytes > 0
    for args in ((0, 10, 8), (4, 1, 8), (4, 33, 8), (4, 10, 0)):
        assert emu.emu_irbpp_dqn_order_log_prob_scratch_bytes(*args) == -1, args
    raw = np.zeros(nbytes + 256, np.uint8)
    scratch = raw.ctypes.data + (-raw.ctypes.data) % 256
    w = IrbppDqnOrderWeights(*([p] * 27 + [ctypes.c_float(0.01)]))
    d = IrbppDqnOrderGrads(*([p] * 21))

    def fwd(atoms=31, B=4, k=10, S=8, stride=1034, lp=p, sf=p, mf=p, acts=a.ctypes.data, sc=scratch, nb=nbytes, ww=w):
        return emu.emu_irbpp_dqn_order_log_prob(ctypes.byref(ww), p, stride, B, k, sf, S, mf, acts, atoms, lp, sc, nb,
                                                None)

    def bwd(atoms=31, g=p, dd=d, dsf=p, dmf=p, nb=nbytes):
        return emu.emu_irbpp_dqn_order_log_prob_backward(ctypes.byref(w), p, 1034, 4, 10, p, 8, p, a.ctypes.data, atoms,
                                                         g, ctypes.byref(dd), dsf, dmf, scratch, nb, None)
    for kw in (dict(atoms=0), dict(atoms=33), dict(B=0), dict(k=1), dict(k=33), dict(S=0), dict(stride=1033),
               dict(lp=None), dict(sf=None), dict(mf=None), dict(acts=None), dict(nb=nbytes - 1), dict(sc=scratch + 4),
               dict(sc=None), dict(ww=IrbppDqnOrderWeights(*([p] * 26 + [None] + [ctypes.c_float(0.01)])))):
        assert fwd(**kw) == IRBPP_EINVAL, kw
    for kw in (dict(atoms=33), dict(g=None), dict(dsf=None), dict(dmf=None), dict(nb=nbytes - 1),
               dict(dd=IrbppDqnOrderGrads(*([p] * 20 + [None])))):
        assert bwd(**kw) == IRBPP_EINVAL, kw
