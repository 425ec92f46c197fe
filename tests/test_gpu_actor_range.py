"""``irbpp_dqn_act`` on the GPU over the whole supported range, through ``DeviceActor`` and through the raw C entry
point, against ``oracle/dqn_port.py`` in float64 on the device.  The cases are those of tests/test_actor_range.py at
1024 bins each: every atom count crossed with every selected_action, every tile-edge n_valid that fits, seeded
networks (full float32 mantissas) in train mode, eval mode and after ``reset_noise()``; a mask apart from column 4,
as float32 and as bool; a wide ``obs_stride``; ``sum_q_map = NULL``; exact ties.

The bar is the accuracy contract of tests/test_actor.py (``Q_RTOL``).  Each group prints its largest scaled error
``|q - q64| / (1 + |q64|)``; the module prints the worst of each group at the end (run with ``-s``)."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from test_actor import check_contract, decode_fixture
from test_actor_range import (ATOMS, MODES, SELS, TIE_FIRSTS, TILE_EDGES, check_ties, col4, dqn_act, make_bins,
                              mask_apart_from_col4, masked, port_q, seeded_net, shape_features, support_for, to_np)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = torch.device("cuda:0")
N = 1024
WORST = {}


@pytest.fixture(scope="module")
def fx():
    return decode_fixture(load_golden("dqn_act"))


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for group, worst in sorted(WORST.items()):
        print("worst scaled error, %s: %.3g" % (group, worst))
    if WORST:
        print("worst scaled error over all groups: %.3g on %s" % (max(WORST.values()), torch.cuda.get_device_name(DEV)))


def record(group, worst):
    WORST[group] = max(WORST.get(group, 0.0), worst)
    return worst


@pytest.mark.parametrize("sel", SELS)
@pytest.mark.parametrize("atoms", ATOMS)
def test_range_on_device(fx, atoms, sel):
    from irbpp_b200 import _lib
    from irbpp_b200.actor import DeviceActor
    case = ATOMS.index(atoms) + SELS.index(sel)
    mode = MODES[case % 3]
    edges = [n for n in TILE_EDGES if n <= sel] + [sel]
    n_valid = [edges[b % len(edges)] for b in range(N)]
    net = seeded_net(sel, atoms, mode).to(DEV)
    obs_np, src = make_bins(fx, sel, n_valid, seed=case)
    sf = shape_features(fx, net, src)
    obs = torch.tensor(obs_np, device=DEV)
    support = torch.tensor(support_for(atoms), device=DEV)
    q64 = port_q(net, obs, sf, support)

    # DeviceActor, the mask as column 4's strided view and no mask
    actor = DeviceActor(net, None, support)
    c4 = col4(obs, sel)
    m = to_np(c4)
    q = to_np(actor.q_values(obs, c4, shape_feature=sf))
    act = to_np(actor.act(obs, c4, shape_feature=sf))
    w_c4 = record("DeviceActor, column-4 mask", check_contract(q, masked(q64, m), act, m))
    qu = to_np(actor.q_values(obs, shape_feature=sf))
    w_none = record("DeviceActor, no mask", check_contract(qu, q64, to_np(actor.act(obs, shape_feature=sf)), None))

    # the raw entry point: rows inside a wider buffer, a contiguous float32 mask apart from column 4, with and
    # without sum_q_map; DeviceActor with the same mask as bool and the same wide rows gives the same bits
    lib = _lib.load()
    L = obs.shape[1]
    wide = torch.full((N, L + 44), float("nan"), device=DEV)
    wide[:, 3:3 + L] = obs
    view = wide[:, 3:3 + L]
    sep = mask_apart_from_col4(m, seed=case)
    sep_t = torch.tensor(sep, device=DEV)
    act_r, q_r = dqn_act(lib, net, view, sel, sf, support, sep_t, prefix="")
    q64s = port_q(net, obs, sf, support, sep_t)
    w_raw = record("raw entry point, separate mask, wide obs_stride", check_contract(q_r, q64s, act_r, sep))
    act_n, _ = dqn_act(lib, net, view, sel, sf, support, sep_t, want_q=False, prefix="")
    assert np.array_equal(act_n, act_r)
    act_nu, _ = dqn_act(lib, net, view, sel, sf, support, None, want_q=False, prefix="")
    assert np.array_equal(act_nu, to_np(actor.act(obs, shape_feature=sf)))
    bool_mask = sep_t == 1
    assert np.array_equal(to_np(actor.q_values(view, bool_mask, shape_feature=sf)), q_r)
    assert np.array_equal(to_np(actor.act(view, bool_mask, shape_feature=sf)), act_r)
    print("atoms %d, sel %d, %s: largest scaled error %.3g (column-4 mask), %.3g (no mask), %.3g (raw, separate mask)"
          % (atoms, sel, mode, w_c4, w_none, w_raw))


@pytest.mark.parametrize("use_mask", [True, False])
def test_ties_on_device(fx, use_mask):
    from irbpp_b200 import _lib
    firsts = (TIE_FIRSTS * (N // len(TIE_FIRSTS) + 1))[:N]
    check_ties(_lib.load(), fx, 500, firsts, use_mask, device=DEV, prefix="")
