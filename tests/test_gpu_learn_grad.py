"""The gradient pass of ``Agent.learn`` at the location level on the GPU: ``irbpp_dqn_log_prob`` /
``irbpp_dqn_log_prob_backward`` on live batches, ``DeviceActor.log_prob`` through autograd, and
``device_learn(..., gradient="device")`` against the reference fixture, against the port's float32 ``learn`` step and
in a training loop.

Bars: the forward and backward bars of ``tests/test_learn_grad.py`` (``3e-6 (1 + |log p64|)``; ``1e-4 max |grad64|``).
Loss: ``loss = -sum_z m_z log p_z`` with ``sum_z m_z = 1`` and ``log p_z <= 0``, so a forward error within
``3e-6 (1 + |log p_z|)`` moves the loss by at most ``3e-6 sum_z m_z (1 + |log p_z|) = 3e-6 (1 + |loss|)``."""
import copy
import types

import numpy as np
import pytest
import torch

from test_gpu_learn_target import (ATOMS, GAMMA, N_STEP, SEL, V_MAX, V_MIN, _FixedBatch, _Recorder,
                                   _SyncFreeOutsideSample, _unchecked, actors, agent_of, clouds_for, features,
                                   filled_bank, nets)
from test_learn_grad import (EMU_RTOL, check_grads, dq_scale, forward_error, log_prob_calls, port_grads)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = torch.device("cuda:0")
LOSS_RTOL = EMU_RTOL                    # 3e-6 (1 + |loss|), derived above


@pytest.fixture(scope="module")
def libs():
    from irbpp_b200 import shapes
    return dict(blockout=shapes.make_blockout_library(32, seed=1),
                general=shapes.make_irregular_library(16, seed=2, num_rotations=8))


@pytest.fixture(scope="module")
def banks(libs):
    return {k: filled_bank(lib, 4096, 8, 3, "location") for k, lib in libs.items()}


@pytest.mark.parametrize("B", [8, 64, 512])
@pytest.mark.parametrize("kind", ["blockout", "general"])
def test_live_batches(libs, banks, kind, B):
    """Forward and backward of the entry points on a sampled batch against the float64 port; a second call gives
    bit-identical outputs."""
    from irbpp_b200 import _lib
    clouds = clouds_for(libs[kind], SEL * 5)
    online, _ = nets("location", clouds)
    _, states, actions, _, _, _, _, _ = banks[kind].sample(B)
    with torch.no_grad():
        sf = online.shape_features_of(states)
        hm = states[:, SEL * 5 + 9:SEL * 5 + 9 + 1024].reshape(-1, 1, 32, 32)
        mf = online.heightEncoder(hm).reshape(states.shape[0], -1)
    g = torch.randn((states.shape[0], ATOMS), device=DEV, generator=torch.Generator(device=DEV).manual_seed(B))
    lib = _lib.load()
    rc, lp, grads = log_prob_calls(lib, online, states, SEL, sf, mf, actions, g, prefix="")
    assert rc == 0
    lp64, ref = port_grads(online, states, sf, mf, actions.cpu().numpy(), g.cpu())
    lp32, ref32 = port_grads(online, states, sf, mf, actions.cpu().numpy(), g.cpu(), dtype=torch.float32)
    err = forward_error(lp, lp64)
    print("%s B %d: |log p - log p64| / (1 + |log p64|) %.3g (torch float32 %.3g), valid rows %d" % (
        kind, B, err, forward_error(lp32, lp64), int((states[:, 4:SEL * 5:5] == 1).sum())))
    assert err <= EMU_RTOL, err
    check_grads(grads, ref, "%s B %d" % (kind, B), dq_scale(lp64, g.cpu().numpy()), ref32)
    rc2, lp2, grads2 = log_prob_calls(lib, online, states, SEL, sf, mf, actions, g, prefix="")
    assert rc2 == 0 and np.array_equal(lp, lp2)
    assert all(np.array_equal(grads[k], grads2[k]) for k in grads)


def test_log_prob_autograd_and_errors(libs, banks):
    """``DeviceActor.log_prob`` differentiates into the module: the shape encoder, the height encoder and the
    NoisyLinear mu / sigma get gradients, and the loss matches the module's own forward.  A state-dict actor and an
    order-level ``device_learn`` are refused; double backward raises."""
    from irbpp_b200.actor import DeviceActor, DeviceOrderActor
    from irbpp_b200.learner_glue import device_learn
    clouds = clouds_for(libs["blockout"], SEL * 5)
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    online, target = nets("location", clouds)
    ref_net = copy.deepcopy(online)
    _, states, actions, _, _, _, weights, _ = banks["blockout"].sample(64)
    actor = DeviceActor(online, clouds, support)
    c0 = clouds.counter
    lp = actor.log_prob(states, actions)
    clouds.counter = c0
    lp_ref = ref_net(states, log=True)[torch.arange(64, device=DEV), actions]
    assert (lp - lp_ref).abs().max().item() <= 1e-5
    g = torch.randn_like(lp)
    (lp * g).sum().backward()
    (lp_ref * g).sum().backward()
    bias_scale = dq_scale(lp_ref.detach().double().cpu().numpy(), g.cpu().numpy())
    for (name, p), (_, q) in zip(online.named_parameters(), ref_net.named_parameters()):
        assert p.grad is not None, name
        scale = q.grad.abs().max().item()
        if name.startswith("fc_z_a.bias"):                  # sum_r da_r = 0: rounding of cancelling terms
            scale = bias_scale * (ref_net.fc_z_a.bias_epsilon.abs().max().item() if "sigma" in name else 1.0)
        assert (p.grad - q.grad).abs().max().item() <= 1e-4 * scale, name
    lp = actor.log_prob(states, actions)
    grad, = torch.autograd.grad(lp.sum(), online.fc_z_a.weight_mu, create_graph=True)
    with pytest.raises(RuntimeError):
        grad.sum().backward()
    with pytest.raises(ValueError):
        DeviceActor(online.state_dict(), clouds, support, train=True).log_prob(states, actions)
    agent = agent_of(online, target, 64)
    with pytest.raises(ValueError, match="location"):
        device_learn(agent, banks["blockout"], DeviceOrderActor.__new__(DeviceOrderActor), None, gradient="device")


class _GradRecorder(_Recorder):
    def log_prob(self, states, actions):
        return self.actor.log_prob(states, actions)


def adam_bar(lr, eps, grad, param):
    """Adam's first step moves a parameter by lr g / (|g| + eps) (m and v bias-corrected to g and g^2); an error d in g
    changes it by at most lr d eps / (|g| + eps)^2 <= lr d / eps, and never by more than 2 lr.  With d = 2e-4 max|g|
    per tensor (the gradient bar, doubled for clip_grad_norm_'s coefficient, which the same errors move), plus one
    float32 ulp of the parameter, the grid both updates are rounded to (fc_z_a.bias's gradient is zero up to
    rounding, so its update is below that ulp)."""
    return lr * min(2.0, 2e-4 * grad.abs().max().item() / eps) + float(np.spacing(np.float32(param.abs().max().item())))


def test_whole_step_matches_the_port_learn(libs, banks):
    """device_learn(gradient="device") against learn_step32 on the same batch, shape features and a*."""
    from oracle.learn_port import learn_step32
    from irbpp_b200.learner_glue import device_learn
    clouds = clouds_for(libs["blockout"], SEL * 5)
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    online, target = nets("location", clouds)
    online_p, target_p = copy.deepcopy(online), copy.deepcopy(target)
    agent = agent_of(online, target, 64)
    lr, eps = agent.optimiser.defaults["lr"], agent.optimiser.defaults["eps"]
    opt_p = torch.optim.Adam(online_p.parameters(), lr=lr, eps=eps)
    on_actor, tg_actor = actors("location", online, target, clouds, support)
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
    sf_t = features("location", tg_actor, clouds, next_states, c0 + 2)
    loss_p, _ = learn_step32(online_p, target_p, opt_p, 10.0, (states, actions, returns, next_states, nonterminals,
                                                               weights), sf_states, sf_t, support, V_MIN, V_MAX,
                             GAMMA ** N_STEP, rec.last)
    dl = ((loss - loss_p).abs() / (1 + loss_p.abs())).max().item()
    assert dl <= 2 * LOSS_RTOL, dl                           # both losses carry float32 forward errors
    worst = 0.0
    for (name, p), q in zip(online.named_parameters(), online_p.parameters()):
        d = (p - q).abs().max().item()
        bar = adam_bar(lr, eps, q.grad, q)
        assert d <= bar, (name, d, bar)
        worst = max(worst, d / lr)
    print("whole step: loss %.3g, largest parameter difference %.3g lr" % (dl, worst))


@pytest.mark.parametrize("case", ["loc_default", "loc_exact"])
def test_reference_fixture_through_device_learn(case):
    """learn.npz (the unmodified reference's Agent.learn) through device_learn(gradient="device"): the loss within
    3e-6 (1 + |loss|) plus the 1e-5 (1 + |loss|) test_learn_golden.py allows the port's float32 step, and the online
    parameters after Adam within 5 % of the learning rate."""
    from irbpp_b200.actor import DeviceActor
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
    clouds = DeviceShapeClouds(points.cpu().numpy(), device=DEV, item_col=SEL * 5)      # one point per shape
    target.reset_noise = lambda: None                       # the fixture holds the noise learn drew
    B = b["states"].shape[0]
    agent = types.SimpleNamespace(online_net=online, target_net=target, batch_size=B, Vmin=v_min, Vmax=v_max,
                                  discount=float(L["discount"]), n=int(L["multi_step"]), norm_clip=clip,
                                  optimiser=torch.optim.Adam(online.parameters(), lr=lr, eps=eps))
    zeros = torch.zeros(B, dtype=torch.int64, device=DEV)
    batch = (zeros, b["states"], b["actions"], b["returns"], b["next_states"], b["nonterminals"], b["weights"], zeros)
    bank = types.SimpleNamespace(sample=lambda n: batch, update_priorities=lambda *a: None)
    loss = device_learn(agent, bank, DeviceActor(online, clouds, support), DeviceActor(target, clouds, support),
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


def test_training_loop_with_device_gradient(libs, banks):
    """20 location iterations: act, step, append, device_learn(gradient="device"), update_target_net every 10, under
    torch's sync check with the exemptions of the existing loop test (sample's error word, reset_noise's host draw);
    the environment's step, which returns its results on the host, is outside the check too."""
    from irbpp_b200.learner_glue import PrioritizedReplayBank, device_learn, get_mask_from_state
    from irbpp_b200.vec_env import GpuVecEnv
    clouds = clouds_for(libs["blockout"], SEL * 5)
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    online, target = nets("location", clouds, seed=3)
    agent = agent_of(online, target, 64)
    on_actor, tg_actor = actors("location", online, target, clouds, support)
    target.reset_noise = _unchecked(target.reset_noise)
    n = 1024
    env = GpuVecEnv(libs["blockout"], None, num_envs=n, device=DEV, item_seed=5)
    state = env.reset().clone()
    bank = PrioritizedReplayBank(n, 40, state.shape[1], DEV, discount=GAMMA, multi_step=N_STEP, seed=5, max_attempts=4096)
    for _ in range(6):                                      # enough transitions for n-step samples
        action = on_actor.act(state, get_mask_from_state(state, SEL))
        nxt = env.step(action)[0]
        bank.append_from_env(env, state, action)
        state = nxt.clone()
    losses = []
    checked = _SyncFreeOutsideSample(bank)
    try:
        torch.cuda.set_sync_debug_mode("error")
        for it in range(20):
            action = on_actor.act(state, get_mask_from_state(state, SEL))
            nxt = _unchecked(lambda a: env.step(a)[0])(action)
            bank.append_from_env(env, state, action)
            state = nxt.clone()
            losses.append(device_learn(agent, checked, on_actor, tg_actor, gradient="device"))
            if (it + 1) % 10 == 0:
                target.load_state_dict(online.state_dict())
    finally:
        torch.cuda.set_sync_debug_mode(0)
    env.close()
    assert all(bool(torch.isfinite(l).all()) for l in losses)
