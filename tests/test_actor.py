"""The location network's act path without a GPU: ``oracle/dqn_port.py`` against the fixture of the unmodified
reference (``tests/golden/dqn_act.npz``), the kernels of ``csrc/irbpp_actor.cuh`` under the host emulator (the header's
host restatement of ``mma.sync`` runs the tensor-core fragments) against the float64 port, the reformulation
of the invalid rows, and ``DeviceActor``'s validation of state dicts.

Accuracy contract (the GPU tests state it too): with ``q64`` the port's expected values in float64 from the same
effective weights, ``|q - q64| <= 1e-4 * (1 + |q64|)`` on every row; the action equals ``argmax q64`` unless the
float64 top-two gap among the unmasked rows is below ``2e-4 * (1 + |max|)``, where any row within that gap is taken;
a fully masked bin acts 0."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.dqn_port import DQNPort

pytestmark = pytest.mark.timeout(900)

SEL = 500
Q_RTOL = 1e-4
GAP_RTOL = 2e-4
P = ctypes.c_void_p


def decode_fixture(d):
    """The compact storage of ``dqn_act.npz`` (tests/golden/make_golden_dqn.py) turned back into the network's 42
    ``state_dict`` arrays (``sd:<key>``, float32) and ``shape_array``: int8 values times a power of two per tensor,
    ``weight_epsilon`` as the float32 outer product of its factors, clouds in steps of 2**-10."""
    d = dict(d)
    for k in [k for k in d if k.startswith("q:")]:
        key = k[2:]
        d["sd:" + key] = d.pop(k).astype(np.float32) * np.float32(2.0 ** int(d.pop("e:" + key)))
    for k in [k for k in d if k.startswith("eps_in:")]:
        layer = k[7:]
        d["sd:%s.weight_epsilon" % layer] = np.outer(d["sd:%s.bias_epsilon" % layer], d.pop(k)).astype(np.float32)
    d["shape_array"] = d.pop("shape_array_q").astype(np.float32) * np.float32(2.0 ** -10)
    return d


@pytest.fixture(scope="module")
def fx():
    return decode_fixture(load_golden("dqn_act"))


def port_from(fx, train, dtype=torch.float64, sel=SEL):
    atoms = fx["sd:fc_z_a.weight_mu"].shape[0]
    net = DQNPort(selected_action=sel, atoms=atoms)
    net.load_state_dict({k[3:]: torch.tensor(v) for k, v in fx.items() if k.startswith("sd:")})
    net.train(train)
    return net.to(dtype)


def shape_features(fx, net):
    """shape_feature of model.py:330-335 from the fixture's point indices (one index set for the whole batch)."""
    obs = fx["obs"]
    items = obs[:, SEL * 5].astype(np.int64)
    pts = torch.tensor(fx["shape_array"][items][:, fx["point_indices"]])
    with torch.no_grad():
        return net.shape_feature(pts.to(next(net.parameters()).dtype))


def check_contract(q, q64, act, mask):
    """The accuracy contract; returns the largest scaled error of q."""
    q64 = np.asarray(q64, np.float64)
    fin = np.isfinite(q64)
    assert np.array_equal(fin, np.isfinite(q)), "masked rows differ"
    err = np.abs(q[fin] - q64[fin]) / (1 + np.abs(q64[fin]))
    worst = float(err.max()) if err.size else 0.0
    assert worst <= Q_RTOL, worst
    for b in range(q64.shape[0]):
        row = np.where(mask[b] == 1, q64[b], -np.inf) if mask is not None else q64[b]
        if not np.isfinite(row).any():
            assert act[b] == 0, b
            continue
        top = row.max()
        within = np.nonzero(row >= top - GAP_RTOL * (1 + abs(top)))[0]
        if len(within) == 1:
            assert act[b] == int(np.argmax(row)), b
        else:
            assert act[b] in within, (b, act[b], within)
    return worst


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_port_reproduces_reference(fx, mode):
    """The port in float32 gives the reference's softmax, sum_q_map and masked actions (float32 tolerance: the
    reference's concat-and-project against the port's, same operations, possibly different kernels)."""
    net = port_from(fx, mode == "train", torch.float32)
    obs = torch.tensor(fx["obs"])
    sf = shape_features(fx, net)
    support = torch.tensor(fx["support"])
    with torch.no_grad():
        q = net(obs, sf)
        sq = (q * support).sum(2)
        act = net.act(obs, sf, support, obs[:, :SEL * 5].reshape(-1, SEL, 5)[:, :, 4])
    np.testing.assert_allclose(q[fx["softmax_rows"]].numpy(), fx[mode + "_softmax"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(sq.numpy(), fx[mode + "_sum_q"], rtol=1e-5, atol=1e-5)
    assert np.array_equal(act.numpy(), fx[mode + "_action"])


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_float32_torch_meets_the_contract(fx, mode):
    """The bar is meaningful: torch's own float32 forward (the reference's arithmetic) meets it against float64."""
    net32, net64 = port_from(fx, mode == "train", torch.float32), port_from(fx, mode == "train", torch.float64)
    obs = torch.tensor(fx["obs"])
    support = torch.tensor(fx["support"])
    mask = obs[:, :SEL * 5].reshape(-1, SEL, 5)[:, :, 4]
    with torch.no_grad():
        sf64 = shape_features(fx, net64)
        q64 = net64.sum_q(obs.double(), sf64, support.double()).numpy()
        q32 = net32.sum_q(obs, sf64.float(), support).numpy()
    act32 = np.where(mask.numpy() == 1, q32, -np.inf).argmax(1)
    worst = check_contract(q32, q64, act32, None)
    print("torch float32 forward: largest |q - q64| / (1 + |q64|) = %.3g" % worst)
    check_contract(np.where(mask.numpy() == 1, q32, -np.inf), np.where(mask.numpy() == 1, q64, -np.inf), act32, mask.numpy())


def test_invalid_row_advantage_is_a0(fx):
    """model.py:347-349 zeroes the embedding of a row with mask != 1; its advantage is then fc_z_a(relu(fc_h_a.bias))
    bit for bit (0 . W + b is exactly b), in both modes and both precisions."""
    for train in (True, False):
        for dtype in (torch.float32, torch.float64):
            net = port_from(fx, train, dtype)
            with torch.no_grad():
                zeros = torch.zeros((3, 128), dtype=dtype)
                w, b = net.fc_h_a.effective()
                assert torch.equal(net.fc_h_a(zeros), b.expand(3, 128)), (train, dtype)      # fc_h_a(0) is its bias
                zero_rows = net.advantage(zeros)
                a0 = net.fc_z_a(torch.relu(b).expand(3, 128))             # the same product on the same input
            assert torch.equal(zero_rows, a0), (train, dtype)


def test_state_dict_validation(fx):
    from irbpp_b200.actor import STATE_DICT_KEYS, check_state_dict
    sd = {k[3:]: torch.tensor(v) for k, v in fx.items() if k.startswith("sd:")}
    assert set(sd) == set(STATE_DICT_KEYS) and len(STATE_DICT_KEYS) == 42
    assert check_state_dict(sd) == 31
    bad = dict(sd); del bad["fc_z_a.bias_epsilon"]
    with pytest.raises(ValueError, match="lacks"):
        check_state_dict(bad)
    bad = dict(sd); bad["project_layer.0.weight"] = torch.zeros(256, 384)
    with pytest.raises(ValueError, match="project_layer.0.weight"):
        check_state_dict(bad)
    bad = dict(sd); bad["fc_h_v.weight_mu"] = torch.zeros(64, 128)      # hidden_size 64: unsupported
    with pytest.raises(ValueError, match="supported"):
        check_state_dict(bad)
    big = DQNPort(atoms=33).state_dict()
    with pytest.raises(ValueError, match="33 atoms"):
        check_state_dict(big)


def test_device_actor_rejects_cpu_tensors(fx):
    from irbpp_b200.actor import DeviceActor
    sd = {k[3:]: torch.tensor(v) for k, v in fx.items() if k.startswith("sd:")}
    with pytest.raises(ValueError, match="CUDA"):
        DeviceActor(sd, None, torch.tensor(fx["support"]))
    with pytest.raises(ValueError, match="module or its state dict"):
        DeviceActor([1, 2], None, torch.tensor(fx["support"]))
    with pytest.raises(ValueError, match="train="):
        DeviceActor(port_from(fx, True, torch.float32), None, torch.tensor(fx["support"]), train=False)


# ---- the kernels under the host emulator ----

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    from test_kernels_emulated import build_emulated
    lib = build_emulated(str(tmp_path_factory.mktemp("emu_actor")))
    lib.emu_irbpp_dqn_scratch_bytes.restype = ctypes.c_int64
    lib.emu_irbpp_dqn_act.restype = ctypes.c_int32
    return lib


def emu_act(lib, net32, obs, sel, sf, support, masked):
    """irbpp_dqn_act on NumPy buffers (host == device under the emulation) with the port's effective weights."""
    from irbpp_b200 import _lib
    from irbpp_b200.actor import _FIELDS
    sd = net32.state_dict()
    eff = {}
    for m in ("fc_h_v", "fc_z_v", "fc_h_a", "fc_z_a"):
        w, b = getattr(net32, m).effective()
        eff[m + ".weight"], eff[m + ".bias"] = w, b
    keep = {f: np.ascontiguousarray((eff[k] if k in eff else sd[k]).detach().numpy(), np.float32) for f, k in _FIELDS}
    w = _lib.IrbppDqnWeights(*([keep[f].ctypes.data for f, _ in _FIELDS] + [ctypes.c_float(0.01)]))
    N = obs.shape[0]
    obs = np.ascontiguousarray(obs, np.float32)
    sf = np.ascontiguousarray(sf, np.float32)
    support = np.ascontiguousarray(support, np.float32)
    nbytes = lib.emu_irbpp_dqn_scratch_bytes(N, sel)
    scratch = np.zeros(nbytes + 256, np.uint8)
    off = (-scratch.ctypes.data) % 256
    actions = np.full(N, -1, np.int64)
    q = np.zeros((N, sel), np.float32)
    rc = lib.emu_irbpp_dqn_act(ctypes.byref(w), P(obs.ctypes.data), ctypes.c_int64(obs.shape[1]), N, sel,
                               P(sf.ctypes.data), P(support.ctypes.data), len(support),
                               P(obs.ctypes.data + 16) if masked else None, ctypes.c_int64(obs.shape[1]), ctypes.c_int64(5),
                               P(actions.ctypes.data), P(q.ctypes.data), P(scratch.ctypes.data + off), ctypes.c_int64(nbytes),
                               None)
    assert rc == 0
    return actions, q


def small_sel(obs, sel):
    """The same bins with only their first sel candidate rows (an observation of selectedAction = sel)."""
    return np.concatenate([obs[:, :sel * 5], obs[:, SEL * 5:]], axis=1)


@pytest.mark.parametrize("sel", [SEL, 24])
def test_emulated_kernels_meet_the_contract(fx, emu, sel):
    """Six fixture bins -- BlockOut mid-episode, truncated (500 valid rows), no-candidate fallback, one valid row, idle,
    and one more BlockOut bin -- through both kernels, in train mode with and without the mask."""
    kinds = fx["kinds"]
    pick = [int(np.nonzero(kinds == k)[0][0]) for k in (0, 1, 2, 3, 4)] + [int(np.nonzero(kinds == 0)[0][5])]
    if sel != SEL:
        pick = pick[:1] + pick[2:]              # 500 valid rows are the same case as 24 at sel = 24
    obs = small_sel(fx["obs"][pick], sel)
    net32, net64 = port_from(fx, True, torch.float32, sel), port_from(fx, True, torch.float64, sel)
    with torch.no_grad():
        items = fx["obs"][pick][:, SEL * 5].astype(np.int64)
        pts = torch.tensor(fx["shape_array"][items][:, fx["point_indices"]])
        sf = net32.shape_feature(pts)
        support = torch.tensor(fx["support"])
        q64 = net64.sum_q(torch.tensor(obs).double(), sf.double(), support.double()).numpy()
    mask = obs[:, :sel * 5].reshape(-1, sel, 5)[:, :, 4]
    for masked in (True, False):
        act, q = emu_act(emu, net32, obs, sel, sf.numpy(), fx["support"], masked)
        want = np.where(mask == 1, q64, -np.inf) if masked else q64
        worst = check_contract(q, want, act, mask if masked else None)
        print("emulated kernels, sel %d, masked %s: largest |q - q64| / (1 + |q64|) = %.3g" % (sel, masked, worst))
