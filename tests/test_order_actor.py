"""The order network's act path without a GPU: ``oracle/order_dqn_port.py`` against the fixture of the unmodified
reference (``tests/golden/dqn_order_act.npz``), ``DeviceOrderActor``'s validation of state dicts, the host mirror of the
order level's point rule, and the kernels of ``csrc/irbpp_order_actor.cuh`` under the host emulator against the
float64 port over ``irbpp_dqn_order_act``'s supported range.

Accuracy contract (``tests/test_actor.py``'s, over the k slots): ``|q - q64| <= 1e-4 * (1 + |q64|)``; the action
equals ``argmax q64`` unless the float64 top-two gap among the unmasked slots is below ``2e-4 * (1 + |max|)``; a fully
masked bin acts 0.  The emulated kernels are also held to ``EMU_RTOL`` (``tests/test_actor_range.py``'s bar): the
slots kernel runs every per-row layer through ``ac_layer``, whose 3xTF32 split that file's mutant builds check."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.order_dqn_port import OrderDQNPort
from test_actor import check_contract
from test_actor_range import EMU_RTOL, MODES, support_for

pytestmark = pytest.mark.timeout(900)

KS = (2, 3, 10, 32)
ATOMS = (1, 31, 32)


def decode_fixture(d):
    """The compact storage of ``dqn_order_act.npz`` (tests/golden/make_golden_order_dqn.py) turned back into the 55
    ``state_dict`` arrays (``sd:<key>``, float32) and the sampled clouds ``clouds`` ``[S, 1024, 3]``."""
    d = dict(d)
    for k in [k for k in d if k.startswith("q:")]:
        key = k[2:]
        d["sd:" + key] = d.pop(k).astype(np.float32) * np.float32(2.0 ** int(d.pop("e:" + key)))
    for k in [k for k in d if k.startswith("eps_in:")]:
        layer = k[7:]
        d["sd:%s.weight_epsilon" % layer] = np.outer(d["sd:%s.bias_epsilon" % layer], d.pop(k)).astype(np.float32)
    d["clouds"] = d.pop("clouds_q").astype(np.float32) * np.float32(2.0 ** -10)
    return d


@pytest.fixture(scope="module")
def fx():
    return decode_fixture(load_golden("dqn_order_act"))


def fixture_sd(fx):
    return {k[3:]: torch.tensor(v) for k, v in fx.items() if k.startswith("sd:")}


def port_from(fx, k, train, dtype=torch.float64):
    net = OrderDQNPort(buffer_size=k, atoms=fx["sd:fc_z_a.weight_mu"].shape[0])
    net.load_state_dict(fixture_sd(fx))
    return net.train(train).to(dtype)


def shape_table(net, clouds):
    """The shape feature of every library shape (model.py:365-372 with the fixture's point indices)."""
    p = next(net.parameters())
    with torch.no_grad():
        return net.shape_feature(torch.as_tensor(clouds).to(p.device, p.dtype))


# ---- the port against the reference ----

@pytest.mark.parametrize("k", [3, 10])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_port_reproduces_reference(fx, k, mode):
    """The port in float32 gives the reference's softmax, sum_q_map and actions (float32 tolerance)."""
    net = port_from(fx, k, mode == "train", torch.float32)
    obs = torch.tensor(fx["obs%d" % k])
    support = torch.tensor(fx["support"])
    sf = shape_table(net, fx["clouds"])
    with torch.no_grad():
        q = net(obs, sf)
        sq = (q * support).sum(2)
    np.testing.assert_allclose(q[fx["softmax_rows"]].numpy(), fx["%s_softmax%d" % (mode, k)], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(sq.numpy(), fx["%s_sum_q%d" % (mode, k)], rtol=1e-5, atol=1e-5)
    assert np.array_equal(net.act(obs, sf, support).numpy(), fx["%s_action%d" % (mode, k)])


@pytest.mark.parametrize("k", [3, 10])
def test_float32_torch_meets_the_contract(fx, k):
    """The bar is meaningful: torch's own float32 forward meets it against float64."""
    for train in (True, False):
        net32, net64 = port_from(fx, k, train, torch.float32), port_from(fx, k, train, torch.float64)
        obs = torch.tensor(fx["obs%d" % k])
        support = torch.tensor(fx["support"])
        with torch.no_grad():
            sf64 = shape_table(net64, fx["clouds"])
            q64 = net64.sum_q(obs.double(), sf64, support.double()).numpy()
            q32 = net32.sum_q(obs, sf64.float(), support).numpy()
        worst = check_contract(q32, q64, q32.argmax(1), None)
        print("k %d, train %s: torch float32 largest scaled error %.3g" % (k, train, worst))


def test_fixture_ids_and_idle_rows(fx):
    """The fixture covers what the kernels must handle: live ids of several shapes and idle all-zero rows."""
    for k in (3, 10):
        obs = fx["obs%d" % k]
        assert (obs[-2:] == 0).all()
        assert len(np.unique(obs[:-2, :k])) > 2 and (obs[:-2, k:] > 0).any()


# ---- validation ----

def test_state_dict_validation(fx):
    from irbpp_b200.actor import ORDER_STATE_DICT_KEYS, STATE_DICT_KEYS, check_order_state_dict
    sd = fixture_sd(fx)
    assert len(sd) == 55 and set(ORDER_STATE_DICT_KEYS) <= set(sd)
    assert set(sd) - set(ORDER_STATE_DICT_KEYS) == {k for k in STATE_DICT_KEYS
                                                    if k.startswith(("init_candidate_embed.", "project_layer."))}
    assert check_order_state_dict(sd) == 31
    bad = dict(sd); del bad["embedder.layers.0.0.module.W_key.weight"]
    with pytest.raises(ValueError, match="order-level DQNBPP"):
        check_order_state_dict(bad)
    bad = dict(sd); bad["gat_project_layer.0.weight"] = torch.zeros(256, 512)
    with pytest.raises(ValueError, match="gat_project_layer.0.weight"):
        check_order_state_dict(bad)
    bad = dict(sd); bad["embedder.layers.0.1.module.0.weight"] = torch.zeros(512, 128)     # feed-forward width 512
    with pytest.raises(ValueError, match="supported"):
        check_order_state_dict(bad)
    with pytest.raises(ValueError, match="33 atoms"):
        check_order_state_dict(OrderDQNPort(atoms=33).state_dict())
    from oracle.dqn_port import DQNPort
    with pytest.raises(ValueError, match="lacks"):                                        # a location network
        check_order_state_dict(DQNPort().state_dict())


def test_device_order_actor_rejects_cpu_tensors(fx):
    from irbpp_b200.actor import DeviceOrderActor
    support = torch.tensor(fx["support"])
    with pytest.raises(ValueError, match="CUDA"):
        DeviceOrderActor(fixture_sd(fx), None, support)
    with pytest.raises(ValueError, match="module or its state dict"):
        DeviceOrderActor([1, 2], None, support)
    with pytest.raises(ValueError, match="train="):
        DeviceOrderActor(port_from(fx, 10, True, torch.float32), None, support, train=False)


def test_order_point_rule_host_mirror():
    """The order level's points: within the first 10 000 points of each cloud, the subsample kept for 1000 acts."""
    from irbpp_b200.pointnet import ORDER_ARRAY_POINTS, ORDER_REDRAW, order_point_indices, pn_indices
    a = order_point_indices(3, 0, 1024, 100000)
    assert a.shape == (1024,) and a.min() >= 0 and a.max() < ORDER_ARRAY_POINTS
    assert order_point_indices(3, 0, 1024, 500).max() < 500
    sub0 = pn_indices(3, 1 << 40, ORDER_ARRAY_POINTS, ORDER_ARRAY_POINTS)                 # epoch 0's subsample
    assert np.array_equal(order_point_indices(3, 7, 1024, 100000), sub0[pn_indices(3, 7, 1024, ORDER_ARRAY_POINTS)])
    assert set(order_point_indices(3, ORDER_REDRAW - 1, 1024, 100000)) <= set(sub0)
    assert not set(order_point_indices(3, ORDER_REDRAW, 1024, 100000)) <= set(sub0)      # redrawn after 1000 acts
    assert not np.array_equal(order_point_indices(3, 1, 1024, 100000), order_point_indices(3, 2, 1024, 100000))


# ---- the kernels under the host emulator ----

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    from irbpp_b200._lib import SIGNATURES
    from test_kernels_emulated import build_emulated
    lib = build_emulated(str(tmp_path_factory.mktemp("emu_order")))
    for name in ("irbpp_dqn_order_act", "irbpp_dqn_order_scratch_bytes"):
        fn = getattr(lib, "emu_" + name)
        fn.restype, fn.argtypes = SIGNATURES[name]
    return lib


def _addr(a):
    return a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data


def _strides(a):
    return tuple(a.stride()) if isinstance(a, torch.Tensor) else tuple(s // a.itemsize for s in a.strides)


def order_act(lib, net32, obs, k, sf, support, mask=None, want_q=True, prefix="emu_"):
    """``irbpp_dqn_order_act`` with every argument explicit: ``obs`` [N, >= k + 1024] (element stride 1, its row stride
    passed as ``obs_stride``), ``sf`` the per-shape table [S, 128], ``mask`` None or float32 [N, k] with its own strides,
    ``want_q=False``: ``sum_q_map = NULL``.  NumPy arrays for the emulated library, CUDA tensors for the real one
    (``prefix=""``).  Weights: the port's effective weights in its mode.  Returns (actions, q or None) as NumPy."""
    from irbpp_b200._lib import IrbppDqnOrderWeights
    from irbpp_b200.actor import _ORDER_FIELDS, NOISY
    dev = obs.device if isinstance(obs, torch.Tensor) else None
    sd = net32.state_dict()
    eff = {k_: sd[k_] for _, k_ in _ORDER_FIELDS if k_ in sd}
    with torch.no_grad():
        for m in NOISY:
            eff[m + ".weight"], eff[m + ".bias"] = getattr(net32, m).effective()
    if dev is None:
        keep = {f: np.ascontiguousarray(eff[k_].detach().cpu().numpy(), np.float32) for f, k_ in _ORDER_FIELDS}
        sf, support = np.ascontiguousarray(sf, np.float32), np.ascontiguousarray(support, np.float32)
    else:
        keep = {f: eff[k_].detach().to(dev, torch.float32).contiguous() for f, k_ in _ORDER_FIELDS}
        sf, support = sf.to(dev, torch.float32).contiguous(), support.to(dev, torch.float32).contiguous()
    w = IrbppDqnOrderWeights(*([_addr(keep[f]) for f, _ in _ORDER_FIELDS] + [ctypes.c_float(0.01)]))
    assert _strides(obs)[1] == 1
    N, S = obs.shape[0], sf.shape[0]
    nbytes = getattr(lib, prefix + "irbpp_dqn_order_scratch_bytes")(N, k, S)
    if dev is None:
        raw = np.zeros(nbytes + 256, np.uint8)
        scratch = raw.ctypes.data + (-raw.ctypes.data) % 256
        actions = np.full(N, -1, np.int64)
        q = np.full((N, k), np.nan, np.float32) if want_q else None
        stream = None
    else:
        raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        scratch = raw.data_ptr() + (-raw.data_ptr()) % 256
        actions = torch.full((N,), -1, dtype=torch.int64, device=dev)
        q = torch.full((N, k), float("nan"), device=dev) if want_q else None
        stream = torch.cuda.current_stream(dev).cuda_stream
    m_row, m_elem = _strides(mask) if mask is not None else (0, 0)
    rc = getattr(lib, prefix + "irbpp_dqn_order_act")(
        ctypes.byref(w), _addr(obs), _strides(obs)[0], N, k, _addr(sf), S, _addr(support), len(support),
        _addr(mask) if mask is not None else None, m_row, m_elem, _addr(actions), _addr(q) if want_q else None,
        scratch, nbytes, stream)
    assert rc == 0, rc
    if dev is not None:
        torch.cuda.synchronize(dev)
        actions, q = actions.cpu(), q.cpu() if want_q else None
    return np.asarray(actions), (np.asarray(q) if want_q else None)


def port_q(net32, obs, sf, support, mask=None, chunk=256):
    """The float64 port's expected values (``-inf`` where ``mask != 1``) from the same parameters, on the device the
    inputs live on."""
    t = lambda a: (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))).double()
    obs, sf, support = t(obs), t(sf), t(support)
    net64 = copy.deepcopy(net32).to(obs.device, torch.float64)
    mask = None if mask is None else t(mask)
    out = []
    with torch.no_grad():
        for i in range(0, obs.shape[0], chunk):
            out.append(net64.sum_q(obs[i:i + chunk], sf, support, None if mask is None else mask[i:i + chunk]).cpu())
    return torch.cat(out).numpy()


def seeded_net(k, atoms, mode, seed=5):
    """Full float32 mantissas (the reference's initialisation rules) in train mode, eval mode, or train mode after a
    second ``reset_noise()``."""
    torch.manual_seed(seed)
    net = OrderDQNPort(buffer_size=k, atoms=atoms)
    if mode == "reset_noise":
        net.reset_noise()
    return net.train(mode != "eval")


def make_obs(fx, k, N, S, seed):
    """N order observations of k slots: the fixture's heightmaps (its idle rows included), ids drawn from [0, S)."""
    rng = np.random.default_rng(seed)
    hm = fx["obs10"][:, 10:]
    src = np.arange(N) % hm.shape[0]
    ids = rng.integers(0, S, (N, k)).astype(np.float32)
    ids[hm[src].max(1) == 0] = 0.0                            # idle bins: all zero
    return np.ascontiguousarray(np.concatenate([ids, hm[src]], axis=1), np.float32)


def emu_contract(q, q64, act, mask):
    worst = check_contract(q, q64, act, mask)
    assert worst <= EMU_RTOL, "largest |q - q64| / (1 + |q64|) = %.3g > EMU_RTOL" % worst
    return worst


def run_case(lib, fx, k, atoms, mode, use_mask, seed=0):
    """Two slots-kernel tiles (the second partial) of bins through the kernels; returns (q, q64, act, mask)."""
    net = seeded_net(k, atoms, mode)
    N = 64 // k + 1
    obs = make_obs(fx, k, N, fx["clouds"].shape[0], seed=k * 7 + atoms)
    sf = shape_table(net, fx["clouds"]).numpy()
    support = support_for(atoms)
    mask = None
    if use_mask:
        rng = np.random.default_rng(seed)
        mask = (rng.random((N, k)) < 0.6).astype(np.float32)
        mask[0] = 0.0                                          # a fully masked bin acts 0
    act, q = order_act(lib, net, obs, k, sf, support, mask)
    q64 = port_q(net, obs, sf, support, mask)
    return q, q64, act, mask


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("atoms", ATOMS)
def test_emulated_range(fx, emu, k, atoms):
    """Every k against every atom count, the mode cycling through train, eval and after reset_noise(), masked for
    odd combinations."""
    i = KS.index(k) + ATOMS.index(atoms)
    mode, use_mask = MODES[i % 3], bool(i % 2)
    q, q64, act, mask = run_case(emu, fx, k, atoms, mode, use_mask)
    worst = emu_contract(q, q64, act, mask)
    print("k %d, atoms %d, %s, masked %s: largest scaled error %.3g" % (k, atoms, mode, use_mask, worst))


@pytest.mark.parametrize("mode", MODES)
def test_emulated_modes_masked_and_unmasked(fx, emu, mode):
    for use_mask in (False, True):
        q, q64, act, mask = run_case(emu, fx, 10, 31, mode, use_mask, seed=1)
        worst = emu_contract(q, q64, act, mask)
        print("k 10, %s, masked %s: largest scaled error %.3g" % (mode, use_mask, worst))


def test_emulated_ties_take_the_first_slot(fx, emu):
    """One atom: every slot's expected value is exactly support[0], so every unmasked slot ties; the action is the
    first unmasked slot, slot 0 unmasked."""
    k = 10
    net = seeded_net(k, 1, "train")
    obs = make_obs(fx, k, 7, fx["clouds"].shape[0], seed=2)
    sf = shape_table(net, fx["clouds"]).numpy()
    support = support_for(1)
    mask = np.zeros((7, k), np.float32)
    firsts = [0, 1, 4, 9, 3, 7, 2]
    for b, f in enumerate(firsts):
        mask[b, f:] = 1.0
        mask[b, f + 1::2] = 0.0
    act, q = order_act(emu, net, obs, k, sf, support, mask)
    assert np.array_equal(q, np.where(mask == 1, support[0], -np.inf))
    assert act.tolist() == firsts
    act, q = order_act(emu, net, obs, k, sf, support)
    assert (q == support[0]).all() and act.tolist() == [0] * 7


def test_emulated_clamped_ids_wide_stride_and_no_sum_q(fx, emu):
    """Ids outside [0, S) are clamped (the reference would raise IndexError), bit for bit the clamped observation;
    rows inside a wider NaN-padded buffer; the action without sum_q_map equals the action with it."""
    k, S = 3, fx["clouds"].shape[0]
    net = seeded_net(k, 31, "eval")
    obs = make_obs(fx, k, 8, S, seed=3)
    obs[1, :3] = [-3.0, S + 5.0, S - 0.5]
    obs[2, :3] = [1e6, -0.9, 2.7]
    clamped = obs.copy()
    clamped[:, :k] = np.clip(np.trunc(obs[:, :k]), 0, S - 1)
    sf = shape_table(net, fx["clouds"]).numpy()
    support = support_for(31)
    wide = np.full((obs.shape[0], obs.shape[1] + 37), np.nan, np.float32)
    wide[:, 5:5 + obs.shape[1]] = obs
    view = wide[:, 5:5 + obs.shape[1]]
    act, q = order_act(emu, net, view, k, sf, support)
    act_c, q_c = order_act(emu, net, clamped, k, sf, support)
    assert np.array_equal(q, q_c) and np.array_equal(act, act_c)
    worst = emu_contract(q, port_q(net, obs, sf, support), act, None)
    act_only, none = order_act(emu, net, view, k, sf, support, want_q=False)
    assert none is None and np.array_equal(act_only, act)
    print("clamped ids, obs_stride %d: largest scaled error %.3g" % (wide.shape[1], worst))


def test_emulated_argument_checks(fx, emu):
    """k, atoms, strides and the scratch outside the supported range are refused with IRBPP_EINVAL."""
    from irbpp_b200._lib import IRBPP_EINVAL, IrbppDqnOrderWeights
    lib = emu
    assert lib.emu_irbpp_dqn_order_scratch_bytes(4, 1, 8) == -1
    assert lib.emu_irbpp_dqn_order_scratch_bytes(4, 33, 8) == -1
    assert lib.emu_irbpp_dqn_order_scratch_bytes(4, 10, 0) == -1
    nbytes = lib.emu_irbpp_dqn_order_scratch_bytes(4, 10, 8)
    assert nbytes > 0
    buf = np.zeros(4096 * 4, np.float32)
    raw = np.zeros(nbytes + 256, np.uint8)
    scratch = raw.ctypes.data + (-raw.ctypes.data) % 256
    w = IrbppDqnOrderWeights(*([buf.ctypes.data] * 27 + [ctypes.c_float(0.01)]))
    acts = np.zeros(4, np.int64)

    def call(k=10, atoms=31, stride=1034, S=8, nb=nbytes, sc=scratch, weights=w):
        return lib.emu_irbpp_dqn_order_act(ctypes.byref(weights), buf.ctypes.data, stride, 4, k, buf.ctypes.data, S,
                                           buf.ctypes.data, atoms, None, 0, 0, acts.ctypes.data, None, sc, nb, None)
    for kw in (dict(k=1), dict(k=33), dict(atoms=0), dict(atoms=33), dict(stride=1033), dict(S=0), dict(nb=nbytes - 1),
               dict(sc=scratch + 4), dict(weights=IrbppDqnOrderWeights(*([buf.ctypes.data] * 26 + [None, 0.01])))):
        assert call(**kw) == IRBPP_EINVAL, kw
