"""``oracle/learn_port.py`` against ``tests/golden/learn.npz``, written by the unmodified reference ``Agent.learn``
(``tests/golden/make_golden_learn.py``): both network levels, the reference's support and an exact grid whose returns
hit the projection's edge cases.

The port's float32 ``learn`` step (``learn_step32``: the reference's torch expressions of ``agent.py:84-121`` on the
port modules, with the fixture's online noise and the target noise ``learn`` drew) reproduces the returned loss and the
priorities within float32 tolerance, and the online parameters after the Adam step within 5 % of the learning rate.
The float64 restatement (``target64``) gives the same loss within ``1e-4 (1 + |loss|)``."""
import copy

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.dqn_port import DQNPort
from oracle.learn_port import distribution, learn_step32, target64
from oracle.order_dqn_port import OrderDQNPort

CASES = ("loc_default", "loc_exact", "order_default", "order_exact")
NOISY = ("fc_h_v", "fc_h_a", "fc_z_v", "fc_z_a")
SEL, K = 500, 10


@pytest.fixture(scope="module")
def gx():
    from test_actor import decode_fixture
    from test_order_actor import decode_fixture as decode_order_fixture
    return dict(learn=dict(load_golden("learn")), loc=decode_fixture(load_golden("dqn_act")),
                order=decode_order_fixture(load_golden("dqn_order_act")))


def case_inputs(gx, case, device="cpu"):
    """The case's online and target port modules (float32, train mode, the fixture's noise and the target noise learn
    drew), its batch, support and constant clouds ``[S, 1, 3]``, all on ``device``."""
    L = gx["learn"]
    level = case.split("_")[0]
    src = gx[level]
    sd = {k[3:]: torch.tensor(v) for k, v in src.items() if k.startswith("sd:")}
    online = (OrderDQNPort(buffer_size=K) if level == "order" else DQNPort(selected_action=SEL))
    online.load_state_dict(sd)
    online = online.to(device).train()
    target = copy.deepcopy(online)
    with torch.no_grad():
        for name in NOISY:
            e_in = torch.tensor(L["%s:tnoise_in:%s" % (case, name)])
            e_out = torch.tensor(L["%s:tnoise_out:%s" % (case, name)])
            getattr(target, name).weight_epsilon.copy_(torch.outer(e_out, e_in))
            getattr(target, name).bias_epsilon.copy_(e_out)
    for p in target.parameters():
        p.requires_grad = False
    obs = src["obs10"] if level == "order" else src["obs"]
    points = (src["clouds"] if level == "order" else src["shape_array"])[:, :1]
    g = lambda k: L["%s:%s" % (case, k)]
    t = lambda a, dt=None: torch.as_tensor(np.asarray(a), dtype=dt, device=device)
    batch = dict(states=t(obs[g("state_rows")]), actions=t(g("actions"), torch.int64), returns=t(g("returns")),
                 next_states=t(obs[g("next_rows")]), nonterminals=t(g("nonterminals")).reshape(-1, 1),
                 weights=t(g("weights")))
    v_min, v_max = float(g("v_min")), float(g("v_max"))
    support = torch.linspace(v_min, v_max, online.atoms, device=device)
    return level, online, target, batch, support, v_min, v_max, t(points)


def shape_features(level, net, points, obs):
    """model.py:330-335 / 365-372 on the constant clouds: per bin at the location level, per shape at the order level."""
    if level == "order":
        return net.shape_feature(points)
    return net.shape_feature(points[obs[:, SEL * 5].long()])


def online_argmax(level, online, points, next_states, support):
    """agent.py:90-92 with the port in float32 (the reference's arithmetic): a* over every row, unmasked."""
    with torch.no_grad():
        sf = shape_features(level, online, points, next_states)
        return (distribution(online, next_states, sf) * support).sum(2).argmax(1)


def constants(gx):
    L = gx["learn"]
    return float(L["discount"]) ** int(L["multi_step"]), float(L["norm_clip"]), float(L["learning_rate"]), float(L["adam_eps"])


@pytest.mark.parametrize("case", CASES)
def test_port_learn_reproduces_reference(gx, case):
    L = gx["learn"]
    gn, clip, lr, eps = constants(gx)
    level, online, target, b, support, v_min, v_max, points = case_inputs(gx, case)
    a_star = online_argmax(level, online, points, b["next_states"], support)
    with torch.no_grad():
        sf_next = shape_features(level, target, points, b["next_states"])
        log_ps_a = distribution(online, b["states"], shape_features(level, online, points, b["states"]), log=True)[
            torch.arange(b["states"].shape[0]), b["actions"]]
    ref64 = target64(None, target, b["next_states"], None, sf_next, support, b["returns"], b["nonterminals"], v_min,
                     v_max, gn, next_actions=a_star, log_ps_a=log_ps_a.numpy())
    opt = torch.optim.Adam(online.parameters(), lr=lr, eps=eps)
    loss, m = learn_step32(online, target, opt, clip, (b["states"], b["actions"], b["returns"], b["next_states"],
                                                       b["nonterminals"], b["weights"]),
                           shape_features(level, online, points, b["states"]), sf_next, support, v_min, v_max, gn, a_star)
    want = L[case + ":loss"]
    np.testing.assert_allclose(loss.numpy(), want, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(loss.numpy(), L[case + ":priorities"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(ref64["loss"], want, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(m.sum(1).numpy(), 1.0, atol=1e-5)
    worst = 0.0
    for key, p in online.named_parameters():
        v = p.detach().numpy().reshape(-1)
        got = v[L["%s:pidx:%s" % (case, key)]]
        worst = max(worst, float(np.abs(got - L["%s:pval:%s" % (case, key)]).max()))
        assert abs(v.astype(np.float64).sum() - float(L["%s:psum:%s" % (case, key)])) <= 0.05 * lr * v.size, key
    assert worst <= 0.05 * lr, worst
    print("%s: |loss - ref| %.3g, float64 |loss - ref| %.3g, largest parameter difference %.3g" % (
        case, np.abs(loss.numpy() - want).max(), np.abs(ref64["loss"] - want).max(), worst))


def test_fixture_covers_the_edge_cases(gx):
    """The exact grid's returns put b on integers (interior, 0, atoms - 1), clamp Tz at both ends, and include terminal
    transitions and blank next states, at both levels."""
    L = gx["learn"]
    from oracle.learn_port import project64
    for case in ("loc_exact", "order_exact"):
        R, nt = L[case + ":returns"], L[case + ":nonterminals"]
        gn = float(L["discount"]) ** int(L["multi_step"])
        pr = project64(np.full((len(R), 31), 1 / 31), R, nt, np.linspace(-15, 15, 31), -15.0, 15.0, gn)
        integer = pr["b"][nt == 0]
        assert {0.0, 30.0} <= set(integer[:, 0]) and (integer[:, 0] == 18.0).any()
        assert (pr["Tz"] == -15.0).all(1).any() and (pr["Tz"] == 15.0).all(1).any()
        level = case.split("_")[0]
        obs = gx[level]["obs10"] if level == "order" else gx[level]["obs"]
        assert (obs[L[case + ":next_rows"]] == 0).all(1).sum() >= 2
