"""The gradient pass of ``Agent.learn`` at the order level on the GPU: ``irbpp_dqn_order_log_prob`` /
``irbpp_dqn_order_log_prob_backward`` on live buffered batches, ``DeviceOrderActor.log_prob`` through autograd,
``device_learn(..., gradient="device")`` at the order level against the port's float32 ``learn`` step and the reference
fixture, ``OrderShapeClouds.sample`` against its host mirror, and the hierarchical loop with the device gradient pass at
both levels.

Bars: those of ``tests/test_order_learn_grad.py`` (``3e-6 (1 + |log p64|)``; ``1e-4 max |grad64|`` or twice torch
float32's own error); the loss bars of ``tests/test_gpu_learn_grad.py``.  The point clouds give every library shape
its own scale and offset: uniform clouds of one size give nearly equal shape features, which makes the slots of a bin
alike and the attention's weight gradients cancel to rounding."""
import copy
import types

import numpy as np
import pytest
import torch

from test_gpu_height_encoder import swap
from test_gpu_learn_grad import LOSS_RTOL, _GradRecorder, adam_bar
from test_gpu_learn_target import (ATOMS, GAMMA, K, N_STEP, SEL, V_MAX, V_MIN, _FixedBatch, _SyncFreeOutsideSample,
                                   _unchecked, actors, agent_of, clouds_for, features, filled_bank, nets)
from test_learn_grad import EMU_RTOL, check_grads, dq_scale, forward_error
from test_order_learn_grad import order_log_prob_calls, order_port_grads

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = torch.device("cuda:0")


def order_clouds(lib, seed=0, points=4096):
    """Clouds whose shapes differ: shape s is uniform in a box of its own size and offset."""
    from irbpp_b200.pointnet import DeviceShapeClouds
    rng = np.random.default_rng(seed)
    S = lib.num_shapes
    scale = rng.uniform(0.05, 1.0, (S, 1, 3))
    offset = rng.uniform(-0.5, 0.5, (S, 1, 3))
    arr = (rng.random((S, points, 3)) * scale + offset).astype(np.float32)
    return DeviceShapeClouds(arr, device=DEV, item_col=K)


@pytest.fixture(scope="module")
def libs():
    from irbpp_b200 import shapes
    return dict(blockout=shapes.make_blockout_library(32, seed=1),
                general=shapes.make_irregular_library(16, seed=2, num_rotations=8))


@pytest.fixture(scope="module")
def banks(libs):
    return {name: filled_bank(lib, 512, 8, 4, "order") for name, lib in libs.items()}


@pytest.mark.parametrize("B", [8, 64, 512])
@pytest.mark.parametrize("kind", ["blockout", "general"])
def test_live_batches(libs, banks, kind, B):
    """Forward and backward of the entry points on a sampled buffered batch against the float64 port; a second call
    gives bit-identical outputs."""
    from irbpp_b200 import _lib
    clouds = order_clouds(libs[kind])
    online, _ = nets("order", clouds)
    _, states, actions, _, _, _, _, _ = banks[kind].sample(B)
    with torch.no_grad():
        sf = online.shape_features_of(states)
        mf = online.heightEncoder(states[:, K:K + 1024].reshape(-1, 1, 32, 32)).reshape(states.shape[0], -1)
    g = torch.randn((states.shape[0], ATOMS), device=DEV, generator=torch.Generator(device=DEV).manual_seed(B))
    lib = _lib.load()
    rc, lp, grads = order_log_prob_calls(lib, online, states, K, sf, mf, actions, g, prefix="")
    assert rc == 0
    lp64, ref = order_port_grads(online, states, sf, mf, actions.cpu().numpy(), g.cpu())
    lp32, ref32 = order_port_grads(online, states, sf, mf, actions.cpu().numpy(), g.cpu(), dtype=torch.float32)
    err = forward_error(lp, lp64)
    print("%s B %d: |log p - log p64| / (1 + |log p64|) %.3g (torch float32 %.3g), distinct ids %d" % (
        kind, B, err, forward_error(lp32, lp64), len(torch.unique(states[:, :K]))))
    assert err <= EMU_RTOL, err
    check_grads(grads, ref, "%s B %d" % (kind, B), dq_scale(lp64, g.cpu().numpy()), ref32)
    rc2, lp2, grads2 = order_log_prob_calls(lib, online, states, K, sf, mf, actions, g, prefix="")
    assert rc2 == 0 and np.array_equal(lp, lp2)
    assert all(np.array_equal(grads[key], grads2[key]) for key in grads)


def test_log_prob_autograd_and_errors(libs, banks):
    """``DeviceOrderActor.log_prob`` differentiates into the module: every named parameter the order network uses gets
    the port module's own gradient (the location level's layers get none in either), and the log-probabilities match
    its forward.  A state-dict actor, double backward and an order actor
    given a location-level batch are refused."""
    from irbpp_b200.actor import DeviceOrderActor
    from irbpp_b200.learner_glue import device_learn
    clouds = order_clouds(libs["blockout"])
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    online, target = nets("order", clouds)
    ref_net = copy.deepcopy(online)
    _, states, actions, _, _, _, _, _ = banks["blockout"].sample(64)
    actor = DeviceOrderActor(online, clouds, support)
    c0 = clouds.counter
    lp = actor.log_prob(states, actions)
    clouds.counter = c0
    lp_ref = ref_net(states, log=True)[torch.arange(64, device=DEV), actions]
    assert (lp - lp_ref).abs().max().item() <= 1e-5
    g = torch.randn_like(lp)
    (lp * g).sum().backward()
    (lp_ref * g).sum().backward()
    bias_scale = dq_scale(lp_ref.detach().double().cpu().numpy(), g.cpu().numpy())
    worst = 0.0
    for (name, p), (_, q) in zip(online.named_parameters(), ref_net.named_parameters()):
        if q.grad is None:                                  # init_candidate_embed, project_layer: the location level's
            assert p.grad is None, name
            continue
        assert p.grad is not None, name
        scale = q.grad.abs().max().item()
        if name.startswith("fc_z_a.bias"):                  # sum_j da_j = 0: rounding of cancelling terms
            scale = bias_scale * (ref_net.fc_z_a.bias_epsilon.abs().max().item() if "sigma" in name else 1.0)
        d = (p.grad - q.grad).abs().max().item()
        assert d <= 1e-4 * scale, (name, d, scale)
        worst = max(worst, d / scale)
    print("log_prob through autograd: largest scaled gradient difference %.3g" % worst)
    lp = actor.log_prob(states, actions)
    grad, = torch.autograd.grad(lp.sum(), online.fc_z_a.weight_mu, create_graph=True)
    with pytest.raises(RuntimeError):
        grad.sum().backward()
    with pytest.raises(ValueError):
        DeviceOrderActor(online.state_dict(), clouds, support, train=True).log_prob(states, actions)
    loc = torch.zeros((64, SEL * 5 + 9 + 1024), device=DEV)
    z = torch.zeros(64, device=DEV)
    bank = types.SimpleNamespace(sample=lambda n: (z.long(), loc, z.long(), z, loc, z[:, None], z + 1, z.long()))
    with pytest.raises(ValueError, match="location"):
        device_learn(agent_of(online, target, 64), bank, actor, None, gradient="device")


def test_whole_step_matches_the_port_learn(libs, banks):
    """device_learn(gradient="device") at the order level against learn_step32 on the same batch, shape features and
    a*: the loss, and every parameter after clip_grad_norm_ and Adam."""
    from oracle.learn_port import learn_step32
    from irbpp_b200.learner_glue import device_learn
    clouds = order_clouds(libs["blockout"])
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    online, target = nets("order", clouds)
    online_p, target_p = copy.deepcopy(online), copy.deepcopy(target)
    agent = agent_of(online, target, 64)
    lr, eps = agent.optimiser.defaults["lr"], agent.optimiser.defaults["eps"]
    opt_p = torch.optim.Adam(online_p.parameters(), lr=lr, eps=eps)
    on_actor, tg_actor = actors("order", online, target, clouds, support)
    rec = _GradRecorder(on_actor)
    batch = banks["blockout"].sample(64)
    _, states, actions, returns, next_states, nonterminals, weights, _ = batch
    c0 = clouds.counter
    torch.manual_seed(11)
    loss = device_learn(agent, _FixedBatch(banks["blockout"], batch), rec, tg_actor, gradient="device")
    torch.manual_seed(11)
    target_p.reset_noise()
    clouds.counter = c0
    sf_states = online_p.shape_features_of(states)
    sf_t = features("order", tg_actor, clouds, next_states, c0 + 2)
    loss_p, _ = learn_step32(online_p, target_p, opt_p, 10.0, (states, actions, returns, next_states, nonterminals,
                                                               weights), sf_states, sf_t, support, V_MIN, V_MAX,
                             GAMMA ** N_STEP, rec.last)
    dl = ((loss - loss_p).abs() / (1 + loss_p.abs())).max().item()
    assert dl <= 2 * LOSS_RTOL, dl
    worst = 0.0
    for (name, p), q in zip(online.named_parameters(), online_p.parameters()):
        d = (p - q).abs().max().item()
        if q.grad is None:                                  # unused at the order level: Adam leaves it alone
            assert d == 0.0, name
            continue
        bar = adam_bar(lr, eps, q.grad, q)
        assert d <= bar, (name, d, bar)
        worst = max(worst, d / lr)
    print("order whole step: loss %.3g, largest parameter difference %.3g lr" % (dl, worst))


@pytest.mark.parametrize("case", ["order_default", "order_exact"])
def test_reference_fixture_through_device_learn(case):
    """learn.npz (the unmodified reference's Agent.learn) at the order level through device_learn(gradient="device"):
    the loss within 3e-6 (1 + |loss|) plus the 1e-5 (1 + |loss|) test_learn_golden.py allows the port's float32 step,
    and the online parameters after Adam within 5 % of the learning rate."""
    from irbpp_b200.actor import DeviceOrderActor
    from irbpp_b200.learner_glue import device_learn
    from irbpp_b200.pointnet import DeviceShapeClouds
    from test_learn_golden import case_inputs, constants
    from conftest import load_golden
    from test_actor import decode_fixture
    from test_order_actor import decode_fixture as decode_order_fixture
    gx = dict(learn=dict(load_golden("learn")), loc=decode_fixture(load_golden("dqn_act")),
              order=decode_order_fixture(load_golden("dqn_order_act")))
    L = gx["learn"]
    gn, clip, lr, eps = constants(gx)
    level, online, target, b, support, v_min, v_max, points = case_inputs(gx, case, DEV)
    clouds = DeviceShapeClouds(points.cpu().numpy(), device=DEV, item_col=K)        # one point per shape
    target.reset_noise = lambda: None                       # the fixture holds the noise learn drew
    B = b["states"].shape[0]
    agent = types.SimpleNamespace(online_net=online, target_net=target, batch_size=B, Vmin=v_min, Vmax=v_max,
                                  discount=float(L["discount"]), n=int(L["multi_step"]), norm_clip=clip,
                                  optimiser=torch.optim.Adam(online.parameters(), lr=lr, eps=eps))
    zeros = torch.zeros(B, dtype=torch.int64, device=DEV)
    batch = (zeros, b["states"], b["actions"], b["returns"], b["next_states"], b["nonterminals"], b["weights"], zeros)
    bank = types.SimpleNamespace(sample=lambda n: batch, update_priorities=lambda *a: None)
    loss = device_learn(agent, bank, DeviceOrderActor(online, clouds, support), DeviceOrderActor(target, clouds, support),
                        gradient="device").detach().cpu().numpy()
    want = L[case + ":loss"]
    err = np.abs(loss - want) / (1 + np.abs(want))
    assert err.max() <= LOSS_RTOL + 1e-5, err.max()
    worst = 0.0
    for key, p in online.named_parameters():
        v = p.detach().cpu().numpy().reshape(-1)
        worst = max(worst, float(np.abs(v[L["%s:pidx:%s" % (case, key)]] - L["%s:pval:%s" % (case, key)]).max()))
        assert abs(v.astype(np.float64).sum() - float(L["%s:psum:%s" % (case, key)])) <= 0.05 * lr * v.size, key
    assert worst <= 0.05 * lr, worst
    print("%s: |loss - reference| / (1 + |loss|) %.3g, largest parameter difference %.3g lr" % (
        case, err.max(), worst / lr))


def test_order_clouds_sample_is_the_point_rule(libs):
    """``OrderShapeClouds.sample`` returns the points of ``order_point_indices`` for its counter, across a subsample
    epoch boundary, and the points ``features`` encodes."""
    from irbpp_b200.pointnet import ORDER_REDRAW, OrderShapeClouds, order_point_indices
    from oracle.dqn_port import DQNPort
    src = clouds_for(libs["blockout"], K, points=12000, seed=4)
    oc = OrderShapeClouds(src)
    ids = torch.tensor([3, 0, 3, src.S - 1], dtype=torch.int32, device=DEV)
    arr = src.shape_array.cpu().numpy()
    for c in (0, 5, ORDER_REDRAW - 1, ORDER_REDRAW, 2 * ORDER_REDRAW + 7):
        got = oc.sample(ids, counter=c).cpu().numpy()
        want = arr[ids.cpu().numpy()][:, order_point_indices(src.seed, c, src.n_points, src.P)]
        assert np.array_equal(got, want), c
    enc = DQNPort().to(DEV).shapeEncoder
    with torch.no_grad():
        f = oc.features(ids, enc, counter=ORDER_REDRAW + 3)
        f_ref = enc(oc.sample(ids, counter=ORDER_REDRAW + 3)).max(1)[0]
    assert (f - f_ref).abs().max().item() <= 1e-5
    c0 = oc.counter
    oc.sample(ids)
    assert oc.counter == c0 + 1


def test_hierarchical_loop_with_device_gradient_at_both_levels(libs):
    """20 iterations of the hierarchical loop on buffered BlockOut bins with DeviceHeightEncoder in all four nets and
    gradient="device" at both levels: order act, candidates, location act, step, append, both device_learn calls,
    update_target_net every 10, under torch's sync check with the existing loop tests' exemptions.  Every loss is
    finite."""
    from irbpp_b200.learner_glue import PrioritizedReplayBank, device_learn, get_mask_from_state
    from irbpp_b200.vec_env import GpuVecEnv
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    n = 1024
    env = GpuVecEnv(libs["blockout"], None, num_envs=n, device=DEV, buffer_size=K, item_seed=5)
    order_state = env.reset().clone()
    levels = {}
    for level, col, width in (("order", K, order_state.shape[1]), ("location", SEL * 5, env.loc_obs_len)):
        clouds = order_clouds(libs["blockout"]) if level == "order" else clouds_for(libs["blockout"], col)
        online, target = nets(level, clouds, seed=3)
        swap(online)
        swap(target)
        target.reset_noise = _unchecked(target.reset_noise)
        bank = PrioritizedReplayBank(n, 40, width, DEV, discount=GAMMA, multi_step=N_STEP, seed=5, max_attempts=4096)
        levels[level] = (agent_of(online, target, 64), bank) + actors(level, online, target, clouds, support)

    def step(state):
        order_actor, loc_actor = levels["order"][2], levels["location"][2]
        order_action = order_actor.act(state)
        loc_state = env.get_action_candidates(order_action, as_tensor=True)
        loc_action = loc_actor.act(loc_state, get_mask_from_state(loc_state, SEL))
        nxt = _unchecked(lambda a: env.step(a)[0])(loc_action)
        levels["order"][1].append_from_env(env, state, order_action)
        levels["location"][1].append_from_env(env, loc_state, loc_action)
        return nxt.clone()
    for _ in range(6):                                      # enough transitions for n-step samples
        order_state = step(order_state)
    losses = []
    try:
        torch.cuda.set_sync_debug_mode("error")
        for it in range(20):
            order_state = step(order_state)
            for level, (agent, bank, on_actor, tg_actor) in levels.items():
                losses.append(device_learn(agent, _SyncFreeOutsideSample(bank), on_actor, tg_actor, gradient="device"))
                if (it + 1) % 10 == 0:
                    agent.target_net.load_state_dict(agent.online_net.state_dict())
    finally:
        torch.cuda.set_sync_debug_mode(0)
    env.close()
    assert len(losses) == 40 and all(bool(torch.isfinite(l).all()) for l in losses)
