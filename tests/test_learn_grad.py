"""The gradient pass of ``Agent.learn`` at the location level without a GPU: ``irbpp_dqn_log_prob`` and
``irbpp_dqn_log_prob_backward`` under the host emulator against the float64 port (``oracle/learn_port.py``,
``distribution(..., log=True)`` with ``torch.autograd``).

Bars: forward ``|log p - log p64| <= EMU_RTOL (1 + |log p64|)`` (``EMU_RTOL = 3e-6``, the emulated act kernels' bar);
backward, for each of the 16 row-section tensors and both feature gradients, ``max |grad - grad64| <= 1e-4 max |grad64|``.
The port runs in float64 from the same effective weights: a NoisyLinear layer in train mode is replaced by an eval-mode
layer whose ``mu`` is the effective tensor, so its ``mu`` gradient is the effective tensor's gradient, and the height
encoder by a constant ``map_feature`` leaf.  torch float32's own error on the same inputs is printed beside the
kernels'."""
import copy
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

from oracle.learn_port import distribution
from test_actor_range import make_bins, seeded_net, shape_features

pytestmark = pytest.mark.timeout(900)

EMU_RTOL = 3e-6
GRAD_RTOL = 1e-4
SELS = (1, 7, 500)
ATOMS = (1, 2, 31, 32)
HM = 32


@pytest.fixture(scope="module")
def fx():
    from test_actor import decode_fixture
    from conftest import load_golden
    return decode_fixture(load_golden("dqn_act"))


def emulated_library(tmp):
    from irbpp_b200._lib import SIGNATURES
    from test_kernels_emulated import build_emulated
    lib = build_emulated(tmp)
    for name in ("irbpp_dqn_log_prob", "irbpp_dqn_log_prob_backward", "irbpp_dqn_log_prob_scratch_bytes"):
        fn = getattr(lib, "emu_" + name)
        fn.restype, fn.argtypes = SIGNATURES[name]
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emulated_library(str(tmp_path_factory.mktemp("emu_learn_grad")))


# ---- the calls ----

def _addr(a):
    return a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data


def row_tensors(net32):
    """The effective row-section tensors of ``net32`` by field of ``irbpp_dqn_grads`` (float32, detached)."""
    from irbpp_b200.actor import NOISY, _ROW_FIELDS
    sd = net32.state_dict()
    eff = {}
    with torch.no_grad():
        for m in NOISY:
            eff[m + ".weight"], eff[m + ".bias"] = getattr(net32, m).effective()
    return {f: (eff[k] if k in eff else sd[k]).detach().float() for f, k in _ROW_FIELDS}


def log_prob_calls(lib, net32, obs, sel, sf, mf, actions, g=None, prefix="emu_"):
    """``irbpp_dqn_log_prob`` and, when ``g`` is given, ``irbpp_dqn_log_prob_backward`` with the port's effective
    weights.  NumPy inputs for the emulated library, CUDA tensors for the real one (``prefix=""``).  Returns
    ``(rc, log_p, grads)`` with ``grads`` a dict field -> array plus ``"shape_feature"`` / ``"map_feature"`` (None
    without ``g``), all NumPy."""
    from irbpp_b200._lib import IrbppDqnGrads, IrbppDqnWeights
    from irbpp_b200.actor import _FIELDS, _ROW_FIELDS
    dev = obs.device if isinstance(obs, torch.Tensor) else None
    ws = row_tensors(net32)
    B, atoms = obs.shape[0], ws["fc_z_a_b"].shape[0]
    if dev is None:
        conv = lambda a, t: np.ascontiguousarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a, t)
        new = lambda shape: np.full(shape, np.nan, np.float32)
        row = obs.strides[0] // 4
    else:
        conv = lambda a, t: torch.as_tensor(a).to(dev, {np.float32: torch.float32, np.int64: torch.int64}[t]).contiguous()
        new = lambda shape: torch.full(shape, float("nan"), device=dev)
        row = obs.stride(0)
    keep = {f: conv(ws[f], np.float32) for f, _ in _ROW_FIELDS}
    sf, mf, a = conv(sf, np.float32), conv(mf, np.float32), conv(actions, np.int64)
    w = IrbppDqnWeights(*([_addr(keep[f]) if f in keep else None for f, _ in _FIELDS] + [ctypes.c_float(0.01)]))
    nbytes = getattr(lib, prefix + "irbpp_dqn_log_prob_scratch_bytes")(B, sel)
    if dev is None:
        raw = np.zeros(nbytes + 256, np.uint8)
        scratch, stream = raw.ctypes.data + (-raw.ctypes.data) % 256, None
    else:
        raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        scratch, stream = raw.data_ptr() + (-raw.data_ptr()) % 256, torch.cuda.current_stream(dev).cuda_stream
    log_p = new((B, atoms))
    rc = getattr(lib, prefix + "irbpp_dqn_log_prob")(ctypes.byref(w), _addr(obs), row, B, sel, _addr(sf), _addr(mf),
                                                     _addr(a), atoms, _addr(log_p), scratch, nbytes, stream)
    grads = None
    if rc == 0 and g is not None:
        gg = conv(g, np.float32)
        out = {f: new(tuple(keep[f].shape)) for f, _ in _ROW_FIELDS}
        out["shape_feature"], out["map_feature"] = new((B, 128)), new((B, 256))
        d = IrbppDqnGrads(*[_addr(out[f]) for f, _ in _ROW_FIELDS])
        rc = getattr(lib, prefix + "irbpp_dqn_log_prob_backward")(
            ctypes.byref(w), _addr(obs), row, B, sel, _addr(sf), _addr(mf), _addr(a), atoms, _addr(gg), ctypes.byref(d),
            _addr(out["shape_feature"]), _addr(out["map_feature"]), scratch, nbytes, stream)
        grads = out
    if dev is not None:
        torch.cuda.synchronize(dev)
        log_p = log_p.cpu()
        grads = None if grads is None else {k: v.cpu() for k, v in grads.items()}
    to_np = lambda x: x.numpy() if isinstance(x, torch.Tensor) else x
    return rc, to_np(log_p), None if grads is None else {k: to_np(v) for k, v in grads.items()}


class _Const(nn.Module):
    """Stands in for the height encoder: returns the ``map_feature`` leaf."""

    def __init__(self, t):
        super().__init__()
        self.t = t

    def forward(self, hm):
        return self.t


def port_grads(net32, obs, sf, mf, actions, g, dtype=torch.float64):
    """``log p(s, a_t, .)`` and the gradients of ``sum(g * log p)`` with respect to the effective row-section tensors
    and both features, by ``torch.autograd`` on the port in ``dtype``, on the device the inputs live on."""
    from irbpp_b200.actor import NOISY, _ROW_FIELDS
    t = lambda a: (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))).to(dtype)
    obs = t(obs)
    dev = obs.device
    eff = row_tensors(net32)
    net = copy.deepcopy(net32).to(dev, dtype)
    with torch.no_grad():
        for m in NOISY:
            getattr(net, m).weight_mu.copy_(eff["%s_w" % m])
            getattr(net, m).bias_mu.copy_(eff["%s_b" % m])
    net.eval()
    sf_leaf = t(sf).to(dev).requires_grad_(True)
    mf_leaf = t(mf).to(dev).requires_grad_(True)
    net.heightEncoder = _Const(mf_leaf)
    B, sel = obs.shape[0], net.sel
    a = torch.as_tensor(np.clip(np.asarray(actions), 0, sel - 1), device=dev)
    lp = distribution(net, obs, sf_leaf, log=True)[torch.arange(B, device=dev), a]
    (lp * t(g).to(dev)).sum().backward()
    params = dict(net.named_parameters())
    out = {}
    for f, k in _ROW_FIELDS:
        name = k.replace(".weight", ".weight_mu").replace(".bias", ".bias_mu") if k.split(".")[0] in NOISY else k
        grad = params[name].grad
        out[f] = np.zeros(tuple(params[name].shape)) if grad is None else grad.detach().cpu().double().numpy()
    out["shape_feature"] = sf_leaf.grad.detach().cpu().double().numpy()
    out["map_feature"] = mf_leaf.grad.detach().cpu().double().numpy()
    return lp.detach().cpu().double().numpy(), out


def forward_error(lp, lp64):
    return float((np.abs(lp.astype(np.float64) - lp64) / (1 + np.abs(lp64))).max())


def grad_errors(grads, ref, bias_scale):
    """max |grad - grad64| / max |grad64| per tensor.  fc_z_a.bias's gradient is sum_r da_r = 0 exactly (the dueling
    combine subtracts the rows' mean advantage), so what remains is rounding of terms that cancel: its scale is
    ``bias_scale``, the size of those terms (sum_b max |dq_b|).  A zero reference (one atom, where log p = 0) takes the
    absolute error."""
    out = {}
    for k, r in ref.items():
        scale = bias_scale if k == "fc_z_a_b" else np.abs(r).max()
        err = np.abs(np.asarray(grads[k], np.float64) - r).max()
        out[k] = float(err / scale) if scale > 0 else float(err)       # one atom: every gradient is exactly 0
    return out


def dq_scale(lp64, g):
    """sum_b max_z |dq_b|, dq = g - softmax(q) sum(g) in float64"""
    g = np.asarray(g, np.float64)
    return float(np.abs(g - np.exp(lp64) * g.sum(1, keepdims=True)).max(1).sum())


def check_grads(grads, ref, label, bias_scale, ref32=None):
    """The gradient bar, GRAD_RTOL, or twice torch float32's own error on the same inputs where that is larger: on
    tens of thousands of rows some pre-activations lie within float32 rounding of zero, where float32 and float64 take
    different sides of a LeakyReLU / ReLU kink; torch float32 then misses GRAD_RTOL too (live general batches of 512:
    1.3e-4 on project_layer.0's weight, 2.1e-4 on shape_feature)."""
    errs = grad_errors(grads, ref, bias_scale)
    e32 = grad_errors(ref32, ref, bias_scale) if ref32 is not None else {}
    for k in ref:
        print("%s %-14s kernel %.3g  torch float32 %s" % (label, k, errs[k], "%.3g" % e32[k] if k in e32 else "-"))
    bad = {k: e for k, e in errs.items() if not e <= max(GRAD_RTOL, 2 * e32.get(k, 0.0))}
    assert not bad, "%s: gradients past the bar: %s" % (label, bad)
    return max(errs.values())


# ---- the inputs ----

def map_features(net32, obs, sel):
    """The height encoder of ``net32`` on the observations' heightmaps (float32): the ``map_feature`` input."""
    B = obs.shape[0]
    hm = torch.from_numpy(np.ascontiguousarray(obs[:, sel * 5 + 9:sel * 5 + 9 + HM * HM])).reshape(B, 1, HM, HM)
    with torch.no_grad():
        return net32.heightEncoder(hm.to(next(net32.parameters()).device)).reshape(B, -1).cpu().numpy()


def grad_case(fx, sel, atoms, mode, n_valid=None, seed=0):
    """Transitions with n_valid 0 (blank), 1, 40 and 103 valid rows (at most sel; 103 of 500 is BlockOut's typical
    count), which puts the batch's compacted rows across several 64-row tiles; a_t: an invalid row of the blank state,
    the one valid row, an invalid row (or the last row), and a row out of range (clamped); g random."""
    net = seeded_net(sel, atoms, mode)
    n_valid = [min(sel, v) for v in (0, 1, 40, 103)] if n_valid is None else list(n_valid)
    obs, src = make_bins(fx, sel, n_valid, seed=sel + atoms + seed)
    obs[0, :sel * 5] = 0.0                                       # a transition without a valid row
    B = obs.shape[0]
    sf = shape_features(fx, net, src).numpy()
    mf = map_features(net, obs, sel)
    rng = np.random.default_rng(seed + 7 * sel + atoms)
    mask = obs[:, 4:sel * 5:5]
    actions = np.zeros(B, np.int64)
    for b in range(B):
        valid, invalid = np.nonzero(mask[b] == 1)[0], np.nonzero(mask[b] != 1)[0]
        pick = (valid if (b % 2 == 1 and len(valid)) or not len(invalid) else invalid)
        actions[b] = rng.choice(pick)
    actions[-1] = sel + 3 if B > 3 else actions[-1]              # out of range: clamped to sel - 1
    g = rng.normal(size=(B, atoms)).astype(np.float32)
    return net, obs, sf, mf, actions, g


# ---- the tests ----

@pytest.mark.parametrize("atoms", ATOMS)
@pytest.mark.parametrize("sel", SELS)
def test_emulated_log_prob_and_backward(fx, emu, sel, atoms):
    for mode in ("train", "eval"):
        net, obs, sf, mf, a, g = grad_case(fx, sel, atoms, mode)
        rc, lp, grads = log_prob_calls(emu, net, obs, sel, sf, mf, a, g)
        assert rc == 0, rc
        lp64, ref = port_grads(net, obs, sf, mf, a, g)
        lp32, ref32 = port_grads(net, obs, sf, mf, a, g, dtype=torch.float32)
        err = forward_error(lp, lp64)
        print("sel %d atoms %d %s: |log p - log p64| / (1 + |log p64|) %.3g (torch float32 %.3g)"
              % (sel, atoms, mode, err, forward_error(lp32, lp64)))
        assert np.isfinite(lp).all() and err <= EMU_RTOL, err
        check_grads(grads, ref, "sel %d atoms %d %s" % (sel, atoms, mode), dq_scale(lp64, g), ref32)


def test_invalid_rows_closed_form(fx, emu):
    """sel 500 with one valid row and with none: the stand-in row carries almost all of fc_z_a's and fc_h_a.bias's
    gradient ((sel - n) copies of -dq / sel), with a_t on the valid row, on an invalid row and out of range."""
    sel, atoms = 500, 31
    net = seeded_net(sel, atoms, "train")
    obs, src = make_bins(fx, sel, [1, 1, 0, 0], seed=11)
    sf = shape_features(fx, net, src).numpy()
    mf = map_features(net, obs, sel)
    mask = obs[:, 4:sel * 5:5]
    one = int(np.nonzero(mask[0] == 1)[0][0])
    a = np.array([one, (one + 1) % sel, 17, -4], np.int64)
    g = np.random.default_rng(3).normal(size=(4, atoms)).astype(np.float32)
    rc, lp, grads = log_prob_calls(emu, net, obs, sel, sf, mf, a, g)
    assert rc == 0
    lp64, ref = port_grads(net, obs, sf, mf, a, g)
    assert forward_error(lp, lp64) <= EMU_RTOL
    check_grads(grads, ref, "sel 500, n_valid 1 / 0", dq_scale(lp64, g))
    for k in ("fc_z_a_w", "fc_h_a_b"):
        assert np.abs(ref[k]).max() > 0


def test_two_runs_are_bit_identical(fx, emu):
    net, obs, sf, mf, a, g = grad_case(fx, 65, 31, "train", n_valid=(0, 1, 65, 65))
    r1 = log_prob_calls(emu, net, obs, 65, sf, mf, a, g)
    r2 = log_prob_calls(emu, net, obs, 65, sf, mf, a, g)
    assert np.array_equal(r1[1], r2[1])
    for k in r1[2]:
        assert np.array_equal(r1[2][k], r2[2][k]), k


def test_argument_checks(emu):
    """atoms 0 and 33, B < 1, sel < 1, a short observation stride, NULL inputs and outputs, a short or misaligned
    scratch are refused with IRBPP_EINVAL."""
    from irbpp_b200._lib import IRBPP_EINVAL, IrbppDqnGrads, IrbppDqnWeights
    buf = np.zeros(1 << 16, np.float32)
    a = np.zeros(4, np.int64)
    p = buf.ctypes.data
    nbytes = emu.emu_irbpp_dqn_log_prob_scratch_bytes(4, 7)
    assert nbytes > 0
    assert emu.emu_irbpp_dqn_log_prob_scratch_bytes(0, 7) == -1 and emu.emu_irbpp_dqn_log_prob_scratch_bytes(4, 0) == -1
    raw = np.zeros(nbytes + 256, np.uint8)
    scratch = raw.ctypes.data + (-raw.ctypes.data) % 256
    w = IrbppDqnWeights(*([p] * 22 + [ctypes.c_float(0.01)]))
    d = IrbppDqnGrads(*([p] * 16))

    def fwd(atoms=31, B=4, sel=7, stride=7 * 5 + 9 + 1024, lp=p, sf=p, acts=a.ctypes.data, sc=scratch, nb=nbytes, ww=w):
        return emu.emu_irbpp_dqn_log_prob(ctypes.byref(ww), p, stride, B, sel, sf, p, acts, atoms, lp, sc, nb, None)

    def bwd(atoms=31, g=p, dd=d, dsf=p, nb=nbytes):
        return emu.emu_irbpp_dqn_log_prob_backward(ctypes.byref(w), p, 7 * 5 + 9 + 1024, 4, 7, p, p, a.ctypes.data,
                                                   atoms, g, ctypes.byref(dd), dsf, p, scratch, nb, None)
    for kw in (dict(atoms=0), dict(atoms=33), dict(B=0), dict(sel=0), dict(stride=7 * 5 + 9 + 1023), dict(lp=None),
               dict(sf=None), dict(acts=None), dict(nb=nbytes - 1), dict(sc=scratch + 4),
               dict(ww=IrbppDqnWeights(*([p] * 21 + [None] + [ctypes.c_float(0.01)])))):
        assert fwd(**kw) == IRBPP_EINVAL, kw
    for kw in (dict(atoms=33), dict(g=None), dict(dsf=None), dict(nb=nbytes - 1),
               dict(dd=IrbppDqnGrads(*([p] * 15 + [None])))):
        assert bwd(**kw) == IRBPP_EINVAL, kw
