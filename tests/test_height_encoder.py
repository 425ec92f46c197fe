"""The height encoder and its backward pass without a GPU: ``irbpp_height_encoder_forward`` /
``irbpp_height_encoder_backward`` under the host emulator against float64 autograd of the port's ``heightEncoder``
(``oracle/dqn_port.py``) with the same weights, and ``DeviceHeightEncoder``'s checks that need no device.

Bars (those of ``tests/test_learn_grad.py``): forward ``|mf - mf64| <= 3e-6 (1 + |mf64|)``; backward, per tensor,
``max |g - g64| <= 1e-4 max |g64|``, or twice torch float32's own error on the same inputs where that is larger (a
pre-activation within float32 rounding of zero takes the other side of a LeakyReLU kink in float32).  torch float32's
own errors are printed beside the kernels'."""
import copy
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

from oracle.dqn_port import DQNPort

pytestmark = pytest.mark.timeout(900)

FWD_RTOL = 3e-6
GRAD_RTOL = 1e-4
HM = 32
FULL_HEIGHT = 0.3            # the default bin's height (bin_dimension z)
FIELDS = (("conv1_w", "conv1.weight"), ("conv1_b", "conv1.bias"), ("conv2_w", "conv2.weight"),
          ("conv2_b", "conv2.bias"), ("conv3_w", "conv3.weight"), ("conv3_b", "conv3.bias"))
NAMES = ("irbpp_height_encoder_forward", "irbpp_height_encoder_backward", "irbpp_height_encoder_scratch_bytes")


@pytest.fixture(scope="module")
def fx():
    from test_actor import decode_fixture
    from conftest import load_golden
    return decode_fixture(load_golden("dqn_act"))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    from irbpp_b200._lib import SIGNATURES
    from test_learn_grad import emulated_library
    lib = emulated_library(str(tmp_path_factory.mktemp("emu_height_encoder")))
    for name in NAMES:
        fn = getattr(lib, "emu_" + name)
        fn.restype, fn.argtypes = SIGNATURES[name]
    return lib


# ---- the calls ----

def _addr(a):
    return a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data


def encoder_calls(lib, seq, rows, col, slope, d_map=None, prefix="emu_"):
    """``irbpp_height_encoder_forward`` and, when ``d_map`` [B, 256] is given, ``irbpp_height_encoder_backward`` on the
    heightmaps at column ``col`` of the observation rows ``rows`` [B, width], read in place (stride = width).  NumPy
    inputs for the emulated library, CUDA tensors for the real one (``prefix=""``).  Returns ``(rc, map [B, 256],
    grads)`` as NumPy, ``grads`` a dict field -> array (None without ``d_map``)."""
    from irbpp_b200._lib import IrbppHeightEncoderGrads, IrbppHeightEncoderWeights
    cuda = isinstance(rows, torch.Tensor)
    B, stride = rows.shape[0], (rows.stride(0) if cuda else rows.strides[0] // 4)
    if cuda:
        dev = rows.device
        keep = {f: getattr_path(seq, k).detach().to(dev, torch.float32).contiguous() for f, k in FIELDS}
        new = lambda shape: torch.full(shape, float("nan"), device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
    else:
        keep = {f: np.ascontiguousarray(getattr_path(seq, k).detach().cpu().numpy(), np.float32) for f, k in FIELDS}
        new = lambda shape: np.full(shape, np.nan, np.float32)
        stream = None
    w = IrbppHeightEncoderWeights(*([_addr(keep[f]) for f, _ in FIELDS] + [ctypes.c_float(slope)]))
    hm = _addr(rows) + 4 * col
    mf = new((B, 256))
    rc = getattr(lib, prefix + "irbpp_height_encoder_forward")(ctypes.byref(w), hm, stride, B, _addr(mf), stream)
    grads = None
    if rc == 0 and d_map is not None:
        nbytes = getattr(lib, prefix + "irbpp_height_encoder_scratch_bytes")(B)
        if cuda:
            dm = torch.as_tensor(d_map).to(dev, torch.float32).contiguous()
            raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
            scratch = raw.data_ptr() + (-raw.data_ptr()) % 256
        else:
            dm = np.ascontiguousarray(d_map, np.float32)
            raw = np.zeros(nbytes + 256, np.uint8)
            scratch = raw.ctypes.data + (-raw.ctypes.data) % 256
        grads = {f: new(tuple(keep[f].shape)) for f, _ in FIELDS}
        d = IrbppHeightEncoderGrads(*[_addr(grads[f]) for f, _ in FIELDS])
        rc = getattr(lib, prefix + "irbpp_height_encoder_backward")(ctypes.byref(w), hm, stride, B, _addr(dm),
                                                                     ctypes.byref(d), scratch, nbytes, stream)
    if cuda:
        torch.cuda.synchronize(dev)
        mf = mf.cpu().numpy()
        grads = None if grads is None else {k: v.cpu().numpy() for k, v in grads.items()}
    return rc, mf, grads


def getattr_path(m, key):
    for part in key.split("."):
        m = getattr(m, part)
    return m


def port_grads(seq, hm, d_map, slope, dtype=torch.float64):
    """The port's ``heightEncoder`` (a copy of ``seq`` with every LeakyReLU at ``slope``) in ``dtype`` on ``hm``
    [B, 1, 32, 32]: the map [B, 256] and the gradients of ``sum(d_map * map)`` by field, NumPy float64."""
    net = copy.deepcopy(seq).to(dtype)
    for m in net:
        if isinstance(m, nn.LeakyReLU):
            m.negative_slope = slope
    hm = torch.as_tensor(hm).to(next(net.parameters()).device, dtype)
    out = net(hm).reshape(hm.shape[0], -1)
    (out * torch.as_tensor(d_map).to(out.device, dtype)).sum().backward()
    grads = {f: getattr_path(net, k).grad.detach().cpu().double().numpy() for f, k in FIELDS}
    return out.detach().cpu().double().numpy(), grads


def forward_error(mf, mf64):
    return float((np.abs(np.asarray(mf, np.float64) - mf64) / (1 + np.abs(mf64))).max())


def grad_errors(grads, ref):
    out = {}
    for k, r in ref.items():
        err, scale = np.abs(np.asarray(grads[k], np.float64) - r).max(), np.abs(r).max()
        out[k] = float(err / scale) if scale > 0 else float(err)
    return out


def check_case(label, mf, grads, mf64, ref, mf32=None, ref32=None):
    """The forward and gradient bars; prints the kernels' errors beside torch float32's."""
    err = forward_error(mf, mf64)
    e32 = forward_error(mf32, mf64) if mf32 is not None else float("nan")
    print("%s: |mf - mf64| / (1 + |mf64|) %.3g (torch float32 %.3g)" % (label, err, e32))
    assert np.isfinite(mf).all() and err <= FWD_RTOL, (label, err)
    if grads is None:
        return
    errs = grad_errors(grads, ref)
    errs32 = grad_errors(ref32, ref) if ref32 is not None else {}
    for k in ref:
        print("%s %-8s kernel %.3g  torch float32 %s" % (label, k, errs[k], "%.3g" % errs32[k] if k in errs32 else "-"))
    bad = {k: e for k, e in errs.items() if not e <= max(GRAD_RTOL, 2 * errs32.get(k, 0.0))}
    assert not bad, "%s: gradients past the bar: %s" % (label, bad)


# ---- the inputs ----

def encoder_of(fx, weights):
    """A reference-shaped ``heightEncoder``: the fixture's reference-initialised tensors, or torch's initialisation
    under a seed."""
    torch.manual_seed(13)
    seq = DQNPort(selected_action=1).heightEncoder
    if weights == "fixture":
        with torch.no_grad():
            for _, k in FIELDS:
                getattr_path(seq, k).copy_(torch.from_numpy(fx["sd:heightEncoder." + k]))
    return seq


def heightmaps(fx, source, B, seed):
    """[B, 1024] float32 heightmaps: the fixture's observations (cycled), uniform in [0, FULL_HEIGHT], all zero (every
    conv1 pre-activation is a bias) or all at the full bin height."""
    if source == "fixture":
        hm = fx["obs"][np.arange(B) % fx["obs"].shape[0], 500 * 5 + 9:]
    elif source == "random":
        hm = np.random.default_rng(seed).uniform(0.0, FULL_HEIGHT, (B, HM * HM))
    elif source == "zeros":
        hm = np.zeros((B, HM * HM))
    else:
        hm = np.full((B, HM * HM), FULL_HEIGHT)
    return np.ascontiguousarray(hm, np.float32)


def observation_rows(hm, sel, seed):
    """Observation rows of width sel * 5 + 9 + 1024 with random candidate rows and item vector, the heightmaps at
    column sel * 5 + 9."""
    B = hm.shape[0]
    rows = np.random.default_rng(seed).uniform(-1.0, 1.0, (B, sel * 5 + 9 + HM * HM)).astype(np.float32)
    rows[:, sel * 5 + 9:] = hm
    return rows


# (heightmap source, B, selected_action) of every weights x slope case
CASES = (("fixture", 7, 500), ("fixture", 64, 1), ("random", 64, 500), ("random", 1, 1), ("zeros", 7, 1),
         ("zeros", 1, 500), ("full", 7, 500), ("full", 64, 1))


# ---- the tests ----

@pytest.mark.parametrize("slope", [0.01, 0.2])
@pytest.mark.parametrize("weights", ["fixture", "seeded"])
def test_emulated_forward_and_backward(fx, emu, weights, slope):
    seq = encoder_of(fx, weights)
    for i, (source, B, sel) in enumerate(CASES):
        hm = heightmaps(fx, source, B, seed=i)
        rows = observation_rows(hm, sel, seed=100 + i)
        d_map = np.random.default_rng(200 + i).normal(size=(B, 256)).astype(np.float32)
        rc, mf, grads = encoder_calls(emu, seq, rows, sel * 5 + 9, slope, d_map)
        assert rc == 0, rc
        hm4 = torch.from_numpy(hm).reshape(B, 1, HM, HM)
        mf64, ref = port_grads(seq, hm4, d_map, slope)
        mf32, ref32 = port_grads(seq, hm4, d_map, slope, dtype=torch.float32)
        check_case("%s slope %g %s B %d sel %d" % (weights, slope, source, B, sel), mf, grads, mf64, ref, mf32, ref32)


def test_backward_of_the_log_prob_map_gradient(fx, emu):
    """d_map = the d_map_feature irbpp_dqn_log_prob_backward returns for a batch (sel 500, 31 atoms, train mode), on
    that batch's heightmaps, read in place from its observation rows."""
    from test_learn_grad import grad_case, log_prob_calls
    sel = 500
    net, obs, sf, mf_in, actions, g = grad_case(fx, sel, 31, "train")
    rc, _, lp_grads = log_prob_calls(emu, net, obs, sel, sf, mf_in, actions, g)
    assert rc == 0
    d_map = lp_grads["map_feature"]
    assert np.abs(d_map).max() > 0
    rc, mf, grads = encoder_calls(emu, net.heightEncoder, obs, sel * 5 + 9, 0.01, d_map)
    assert rc == 0
    B = obs.shape[0]
    hm4 = torch.from_numpy(np.ascontiguousarray(obs[:, sel * 5 + 9:])).reshape(B, 1, HM, HM)
    mf64, ref = port_grads(net.heightEncoder, hm4, d_map, 0.01)
    mf32, ref32 = port_grads(net.heightEncoder, hm4, d_map, 0.01, dtype=torch.float32)
    assert forward_error(mf_in, mf64) <= FWD_RTOL          # the map the log-prob call took (torch float32)
    check_case("log-prob d_map", mf, grads, mf64, ref, mf32, ref32)


def test_two_runs_are_bit_identical(fx, emu):
    seq = encoder_of(fx, "seeded")
    hm = heightmaps(fx, "random", 40, seed=3)
    rows = observation_rows(hm, 7, seed=4)
    d_map = np.random.default_rng(5).normal(size=(40, 256)).astype(np.float32)
    r1 = encoder_calls(emu, seq, rows, 7 * 5 + 9, 0.01, d_map)
    r2 = encoder_calls(emu, seq, rows, 7 * 5 + 9, 0.01, d_map)
    assert r1[0] == 0 and r2[0] == 0
    assert np.array_equal(r1[1], r2[1])
    for k in r1[2]:
        assert np.array_equal(r1[2][k], r2[2][k]), k


def test_argument_checks(emu):
    """B < 1, NULL inputs, weights and outputs, a negative or non-finite slope, a heightmap stride below 1024 and a
    short or misaligned scratch are refused with IRBPP_EINVAL; scratch_bytes(0) is -1."""
    from irbpp_b200._lib import IRBPP_EINVAL, IrbppHeightEncoderGrads, IrbppHeightEncoderWeights
    buf = np.zeros(1 << 16, np.float32)
    p = buf.ctypes.data
    assert emu.emu_irbpp_height_encoder_scratch_bytes(0) == -1
    assert emu.emu_irbpp_height_encoder_scratch_bytes(-3) == -1
    nbytes = emu.emu_irbpp_height_encoder_scratch_bytes(2)
    assert nbytes >= 2 * 9652 * 4
    raw = np.zeros(nbytes + 256, np.uint8)
    scratch = raw.ctypes.data + (-raw.ctypes.data) % 256
    W = lambda slope=0.01, null=None: IrbppHeightEncoderWeights(*([None if i == null else p for i in range(6)] +
                                                                  [ctypes.c_float(slope)]))
    G = lambda null=None: IrbppHeightEncoderGrads(*[None if i == null else p for i in range(6)])

    def fwd(w=None, hm=p, stride=1024, B=2, out=p):
        return emu.emu_irbpp_height_encoder_forward(None if w is False else ctypes.byref(w or W()), hm, stride, B, out,
                                                    None)

    def bwd(w=None, hm=p, stride=1024, B=2, dm=p, g=None, sc=scratch, nb=nbytes):
        return emu.emu_irbpp_height_encoder_backward(None if w is False else ctypes.byref(w or W()), hm, stride, B, dm,
                                                     None if g is False else ctypes.byref(g or G()), sc, nb, None)
    assert fwd() == 0 and bwd() == 0                    # zeros: the calls themselves are valid
    bad_weights = [W(slope=-0.01), W(slope=float("nan")), W(slope=float("inf"))] + [W(null=i) for i in range(6)]
    for kw in [dict(B=0), dict(B=-1), dict(hm=None), dict(w=False), dict(stride=1023), dict(out=None)] + \
            [dict(w=w) for w in bad_weights]:
        assert fwd(**kw) == IRBPP_EINVAL, kw
    for kw in [dict(B=0), dict(hm=None), dict(w=False), dict(stride=1023), dict(dm=None), dict(g=False), dict(sc=None),
               dict(nb=nbytes - 1), dict(sc=scratch + 4)] + [dict(w=w) for w in bad_weights] + \
            [dict(g=G(null=i)) for i in range(6)]:
        assert bwd(**kw) == IRBPP_EINVAL, kw


def test_module_checks_without_a_device():
    """DeviceHeightEncoder takes the reference's Sequential and keeps its children and parameters; any other structure,
    mixed or negative slopes, and a CPU input raise ValueError."""
    from irbpp_b200.height_encoder import DeviceHeightEncoder
    net = DQNPort(selected_action=3)
    seq = net.heightEncoder
    params = dict(seq.named_parameters())
    enc = DeviceHeightEncoder(seq)
    assert all(a is b for a, b in zip(enc.children(), seq.children()))
    assert all(params[n] is p for n, p in enc.named_parameters()) and len(params) == 6
    keys = list(net.state_dict())
    net.heightEncoder = enc
    assert list(net.state_dict()) == keys
    with pytest.raises(ValueError):
        enc(torch.zeros(2, 1, HM, HM))
    assert not DeviceHeightEncoder(copy.deepcopy(seq).eval()).training

    def variant(edit):
        s = copy.deepcopy(seq)
        edit(s)
        return s
    bad = [
        nn.Sequential(*list(seq.children())),                                        # unnamed children
        variant(lambda s: setattr(s, "conv2", nn.Conv2d(16, 32, 4, stride=1, padding=1))),
        variant(lambda s: setattr(s, "conv3", nn.Conv2d(32, 8, 3, stride=1, padding=1))),
        variant(lambda s: setattr(s, "conv1", nn.Conv2d(1, 16, 4, stride=2, padding=1, bias=False))),
        variant(lambda s: setattr(s, "conv1", nn.Conv2d(1, 16, 4, stride=2, padding=1, padding_mode="reflect"))),
        variant(lambda s: setattr(s, "relu2", nn.ReLU())),
        variant(lambda s: setattr(s, "relu3", nn.LeakyReLU(0.2))),
        variant(lambda s: [setattr(getattr(s, r), "negative_slope", -0.01) for r in ("relu1", "relu2", "relu3")]),
        variant(lambda s: [setattr(getattr(s, r), "negative_slope", float("nan")) for r in ("relu1", "relu2", "relu3")]),
        variant(lambda s: s.add_module("extra", nn.Identity())),
        nn.ModuleList(list(seq.children())),
    ]
    for s in bad:
        with pytest.raises(ValueError):
            DeviceHeightEncoder(s)
    # a common slope other than the default is accepted
    DeviceHeightEncoder(variant(lambda s: [setattr(getattr(s, r), "negative_slope", 0.2) for r in ("relu1", "relu2", "relu3")]))
