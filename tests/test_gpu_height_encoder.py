"""The height encoder on the GPU: ``irbpp_height_encoder_forward`` / ``irbpp_height_encoder_backward`` on live batches,
``DeviceHeightEncoder`` as a drop-in for both network levels' ``heightEncoder``, and ``device_learn`` with it swapped
into the online net, against the port's float32 learn step, against the reference fixture and in the hierarchical
training loop.

Bars: those of ``tests/test_height_encoder.py`` (forward ``3e-6 (1 + |mf64|)``; per gradient tensor ``1e-4 max |g64|``
or twice torch float32's own error) and, for whole learn steps, those of ``tests/test_gpu_learn_grad.py``.  torch's
float32 convolutions are evaluated with cudnn off, the reference's default training mode: cudnn would run them in
TF32."""
import copy
import io
import types

import numpy as np
import pytest
import torch

from test_gpu_learn_grad import LOSS_RTOL, _GradRecorder, adam_bar
from test_gpu_learn_target import (ATOMS, GAMMA, K, N_STEP, SEL, V_MAX, V_MIN, _FixedBatch, _Recorder,
                                   _SyncFreeOutsideSample, _unchecked, actors, agent_of, clouds_for, features,
                                   filled_bank, nets)
from test_height_encoder import FWD_RTOL, HM, check_case, encoder_calls, forward_error, port_grads

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def libs():
    from irbpp_b200 import shapes
    return dict(blockout=shapes.make_blockout_library(32, seed=1),
                general=shapes.make_irregular_library(16, seed=2, num_rotations=8))


@pytest.fixture(scope="module")
def banks(libs):
    return {k: filled_bank(lib, 4096, 8, 3, "location") for k, lib in libs.items()}


@pytest.fixture(scope="module")
def order_bank(libs):
    return filled_bank(libs["blockout"], 512, 10, 4, "order")


def swap(net):
    from irbpp_b200.height_encoder import DeviceHeightEncoder
    net.heightEncoder = DeviceHeightEncoder(net.heightEncoder)
    return net


def heightmaps_of(states, col):
    return states[:, col:col + HM * HM].reshape(-1, 1, HM, HM)


@pytest.mark.parametrize("B", [8, 64, 512, 4096])
@pytest.mark.parametrize("kind", ["blockout", "general"])
def test_live_batches(libs, banks, kind, B):
    """Forward and backward on the heightmaps of a sampled batch, read in place from the observation rows, against
    float64 autograd; a second call gives bit-identical outputs."""
    from irbpp_b200 import _lib
    clouds = clouds_for(libs[kind], SEL * 5)
    online, _ = nets("location", clouds)
    _, states, _, _, _, _, _, _ = banks[kind].sample(B)
    B = states.shape[0]
    d_map = torch.randn((B, 256), device=DEV, generator=torch.Generator(device=DEV).manual_seed(B))
    lib = _lib.load()
    rc, mf, grads = encoder_calls(lib, online.heightEncoder, states, SEL * 5 + 9, 0.01, d_map, prefix="")
    assert rc == 0
    hm = heightmaps_of(states, SEL * 5 + 9)
    mf64, ref = port_grads(online.heightEncoder, hm, d_map, 0.01)
    with torch.backends.cudnn.flags(enabled=False):
        mf32, ref32 = port_grads(online.heightEncoder, hm, d_map, 0.01, dtype=torch.float32)
    check_case("%s B %d" % (kind, B), mf, grads, mf64, ref, mf32, ref32)
    rc2, mf2, grads2 = encoder_calls(lib, online.heightEncoder, states, SEL * 5 + 9, 0.01, d_map, prefix="")
    assert rc2 == 0 and np.array_equal(mf, mf2)
    assert all(np.array_equal(grads[k], grads2[k]) for k in grads)


@pytest.mark.parametrize("level", ["location", "order"])
def test_drop_in(libs, banks, order_bank, level):
    """After the swap: the same Parameter objects, the same state_dict keys and values; deepcopy and a torch.save /
    torch.load round trip work; the device actors act as on the original; the module's output is the original's
    within the forward bar, also through autograd; bad inputs raise ValueError."""
    from irbpp_b200.height_encoder import DeviceHeightEncoder
    col = K if level == "order" else SEL * 5
    clouds = clouds_for(libs["blockout"], col)
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    net, _ = nets(level, clouds)
    orig = copy.deepcopy(net)
    params = list(net.named_parameters())
    sd = net.state_dict()
    swap(net)
    assert [(n, id(p)) for n, p in net.named_parameters()] == [(n, id(p)) for n, p in params]
    sd2 = net.state_dict()
    assert list(sd2) == list(sd) and all(torch.equal(sd[k], sd2[k]) for k in sd)
    bank = order_bank if level == "order" else banks["blockout"]
    states = bank.sample(64)[1]
    hm = heightmaps_of(states, col + (0 if level == "order" else 9))
    with torch.no_grad():
        mf64 = copy.deepcopy(orig.heightEncoder).double()(hm.double()).reshape(64, -1).cpu().numpy()
        with torch.backends.cudnn.flags(enabled=False):
            ref = orig.heightEncoder(hm).reshape(64, -1).cpu().numpy()
        got = net.heightEncoder(hm)
    assert tuple(got.shape) == (64, 4, 8, 8)
    got = got.reshape(64, -1).cpu().numpy()
    print("%s: |mf - mf64| / (1 + |mf64|) %.3g (torch float32 %.3g)" % (level, forward_error(got, mf64),
                                                                        forward_error(ref, mf64)))
    assert forward_error(got, mf64) <= FWD_RTOL
    with torch.no_grad():
        assert np.array_equal(net.heightEncoder(hm.contiguous().clone()).reshape(64, -1).cpu().numpy(), got)
        assert np.array_equal(net.heightEncoder(hm.transpose(2, 3).contiguous().transpose(2, 3)).reshape(64, -1)
                              .cpu().numpy(), got)                     # a non-contiguous layout is copied first
    # copies
    for other in (copy.deepcopy(net).heightEncoder, _round_trip(net.heightEncoder)):
        assert isinstance(other, DeviceHeightEncoder)
        with torch.no_grad():
            assert np.array_equal(other(hm).reshape(64, -1).cpu().numpy(), got)
    # the device actors read the same weights
    A = actors(level, net, net, clouds, support)[0]
    A0 = actors(level, orig, orig, clouds, support)[0]
    c0 = clouds.counter
    kw = "shape_features" if level == "order" else "shape_feature"
    sf = features(level, A0, clouds, states, c0)
    assert torch.equal(A.act(states, **{kw: sf}), A0.act(states, **{kw: sf}))
    # autograd reaches every conv parameter
    out = net.heightEncoder(hm)
    out.sum().backward()
    assert all(p.grad is not None for p in net.heightEncoder.parameters())
    # input checks
    enc = net.heightEncoder
    for bad in (hm.double(), hm[:, :, :16], hm.reshape(64, 1024), hm.clone().requires_grad_(True), hm.cpu()):
        with pytest.raises(ValueError):
            enc(bad)
    with pytest.raises(ValueError):
        copy.deepcopy(enc).cpu()(hm)                                   # weights on another device


def _round_trip(module):
    buf = io.BytesIO()
    torch.save(module, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=False)


@pytest.mark.parametrize("level,gradient", [("location", "device"), ("location", "torch"), ("order", "torch")])
def test_device_learn_matches_the_port_learn(libs, banks, order_bank, level, gradient):
    """device_learn with the encoder swapped into the online net against learn_step32 on the same batch, shape
    features and a* (the port with torch's convolutions, cudnn off): the loss within 2 LOSS_RTOL (1 + |loss|) and the
    parameters after Adam within adam_bar."""
    from oracle.learn_port import learn_step32
    from irbpp_b200.learner_glue import device_learn
    bank = order_bank if level == "order" else banks["blockout"]
    clouds = clouds_for(libs["blockout"], K if level == "order" else SEL * 5)
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    online, target = nets(level, clouds)
    online_p, target_p = copy.deepcopy(online), copy.deepcopy(target)
    swap(online)
    agent = agent_of(online, target, 64)
    lr, eps = agent.optimiser.defaults["lr"], agent.optimiser.defaults["eps"]
    opt_p = torch.optim.Adam(online_p.parameters(), lr=lr, eps=eps)
    on_actor, tg_actor = actors(level, online, target, clouds, support)
    rec = (_GradRecorder if gradient == "device" else _Recorder)(on_actor)
    batch = bank.sample(64)
    _, states, actions, returns, next_states, nonterminals, weights, _ = batch
    c0 = clouds.counter
    torch.manual_seed(11)
    loss = device_learn(agent, _FixedBatch(bank, batch), rec, tg_actor, gradient=gradient)
    torch.manual_seed(11)
    target_p.reset_noise()
    clouds.counter = c0
    with torch.backends.cudnn.flags(enabled=False):
        sf_states = online_p.shape_features_of(states)
        sf_t = features(level, tg_actor, clouds, next_states, c0 + 2)
        loss_p, _ = learn_step32(online_p, target_p, opt_p, 10.0, (states, actions, returns, next_states, nonterminals,
                                                                   weights), sf_states, sf_t, support, V_MIN, V_MAX,
                                 GAMMA ** N_STEP, rec.last)
    dl = ((loss - loss_p).abs() / (1 + loss_p.abs())).max().item()
    assert dl <= 2 * LOSS_RTOL, dl
    worst = 0.0
    for (name, p), q in zip(online.named_parameters(), online_p.parameters()):
        d = (p - q).abs().max().item()
        bar = adam_bar(lr, eps, q.grad, q) if q.grad is not None else 0.0      # unused at the order level: unchanged
        assert d <= bar, (name, d, bar)
        worst = max(worst, d / lr)
    print("%s gradient=%s: loss %.3g, largest parameter difference %.3g lr" % (level, gradient, dl, worst))


@pytest.mark.parametrize("case", ["loc_default", "loc_exact", "order_default", "order_exact"])
def test_reference_fixture_through_device_learn(case):
    """learn.npz (the unmodified reference's Agent.learn) through device_learn with the encoder swapped into the
    online net (location: gradient="device"; order: the module's own forward): the loss within 3e-6 (1 + |loss|) plus
    1e-5 (1 + |loss|), and the online parameters after Adam within 5 % of the learning rate."""
    from irbpp_b200.actor import DeviceActor, DeviceOrderActor
    from irbpp_b200.learner_glue import device_learn
    from irbpp_b200.pointnet import DeviceShapeClouds
    from oracle.learn_port import ReferenceOrderDQN
    from test_learn_golden import case_inputs, constants
    from conftest import load_golden
    from test_actor import decode_fixture
    from test_order_actor import decode_fixture as decode_order_fixture
    gx = dict(learn=dict(load_golden("learn")), loc=decode_fixture(load_golden("dqn_act")),
              order=decode_order_fixture(load_golden("dqn_order_act")))
    L = gx["learn"]
    gn, clip, lr, eps = constants(gx)
    level, online, target, b, support, v_min, v_max, points = case_inputs(gx, case, DEV)
    clouds = DeviceShapeClouds(points.cpu().numpy(), device=DEV, item_col=K if level == "order" else SEL * 5)
    if level == "order":                  # modules whose forward samples the clouds, as the reference's does
        online_r, target_r = [ReferenceOrderDQN(clouds, buffer_size=K, atoms=online.atoms).to(DEV).train()
                              for _ in range(2)]
        online_r.load_state_dict(online.state_dict())
        target_r.load_state_dict(target.state_dict())
        for p in target_r.parameters():
            p.requires_grad = False
        online, target = online_r, target_r
    swap(online)
    target.reset_noise = lambda: None                       # the fixture holds the noise learn drew
    B = b["states"].shape[0]
    agent = types.SimpleNamespace(online_net=online, target_net=target, batch_size=B, Vmin=v_min, Vmax=v_max,
                                  discount=float(L["discount"]), n=int(L["multi_step"]), norm_clip=clip,
                                  optimiser=torch.optim.Adam(online.parameters(), lr=lr, eps=eps))
    zeros = torch.zeros(B, dtype=torch.int64, device=DEV)
    batch = (zeros, b["states"], b["actions"], b["returns"], b["next_states"], b["nonterminals"], b["weights"], zeros)
    bank = types.SimpleNamespace(sample=lambda n: batch, update_priorities=lambda *a: None)
    A = DeviceOrderActor if level == "order" else DeviceActor
    loss = device_learn(agent, bank, A(online, clouds, support), A(target, clouds, support),
                        gradient="torch" if level == "order" else "device").detach().cpu().numpy()
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


def test_hierarchical_loop_with_device_encoders(libs):
    """20 iterations of the hierarchical loop on buffered BlockOut bins with the encoder swapped into all four nets:
    order act, candidates, location act, step, append, both device_learn calls (location gradient="device"),
    update_target_net every 10, under torch's sync check with the existing loop tests' exemptions (sample's error
    word, reset_noise's host draw, the environment's step).  Every loss is finite."""
    from irbpp_b200.learner_glue import PrioritizedReplayBank, device_learn, get_mask_from_state
    from irbpp_b200.vec_env import GpuVecEnv
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    n = 1024
    env = GpuVecEnv(libs["blockout"], None, num_envs=n, device=DEV, buffer_size=K, item_seed=5)
    order_state = env.reset().clone()
    levels = {}
    for level, col, width in (("order", K, order_state.shape[1]), ("location", SEL * 5, env.loc_obs_len)):
        clouds = clouds_for(libs["blockout"], col)
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
                losses.append(device_learn(agent, _SyncFreeOutsideSample(bank), on_actor, tg_actor,
                                           gradient="device" if level == "location" else "torch"))
                if (it + 1) % 10 == 0:
                    agent.target_net.load_state_dict(agent.online_net.state_dict())
    finally:
        torch.cuda.set_sync_debug_mode(0)
    env.close()
    assert len(losses) == 40 and all(bool(torch.isfinite(l).all()) for l in losses)
