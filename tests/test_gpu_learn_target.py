"""The target half of ``Agent.learn`` on the GPU: ``DeviceActor.target`` / ``DeviceOrderActor.target`` on batches a
``PrioritizedReplayBank`` fed by live ``GpuVecEnv`` bins returns, against the float64 port on the device and against
torch's own float32 ``agent.py:100-115``; ``learner_glue.device_learn`` against the port's float32 torch ``learn``; and
the hierarchical loop with both ``device_learn`` calls.

Bars (``tests/test_learn_target.py``'s, with the GPU's looser p bar): ``|p - p64| <= 1e-5``; ``sum |m - m64| <= sum
|p - p64| + 2 max |b - b64| + 1e-6``; ``|m - m_torch| <= 1e-6`` where ``m_torch`` is the reference's float32 expression
evaluated on the device from the kernel's ``p`` (its ``index_add_`` adds in no fixed order, hence a tolerance)."""
import copy
import types

import numpy as np
import pytest
import torch

from oracle.learn_port import (ReferenceDQN, ReferenceOrderDQN, distribution, learn_step32, target64,
                               torch_projection)
from test_actor import check_contract

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = torch.device("cuda:0")
SEL, K, ATOMS = 500, 10, 31
V_MIN, V_MAX, GAMMA, N_STEP = -1.0, 8.0, 0.99, 3


def clouds_for(lib, item_col, points=4096, seed=0):
    from irbpp_b200.pointnet import DeviceShapeClouds
    arr = np.random.default_rng(seed).random((lib.num_shapes, points, 3)).astype(np.float32) * 0.1
    return DeviceShapeClouds(arr, device=DEV, item_col=item_col)


def filled_bank(lib, n, steps, seed, level):
    """A PrioritizedReplayBank of n memories fed by ``steps`` steps of n live bins (random valid actions; at the order
    level random slots), as trainer.py:181-186 appends."""
    from irbpp_b200.learner_glue import PrioritizedReplayBank, get_mask_from_state
    from irbpp_b200.vec_env import GpuVecEnv
    k = K if level == "order" else 1
    env = GpuVecEnv(lib, None, num_envs=n, device=DEV, buffer_size=k, item_seed=seed)
    state = env.reset().clone()
    bank = PrioritizedReplayBank(n, steps + 4, state.shape[1], DEV, discount=GAMMA, multi_step=N_STEP, seed=seed,
                                 max_attempts=4096)
    gen = torch.Generator(device=DEV); gen.manual_seed(seed)
    for _ in range(steps):
        if level == "order":
            action = torch.randint(0, k, (n,), device=DEV, generator=gen)
            loc = env.get_action_candidates(action, as_tensor=True)
        else:
            loc = state
        q = torch.rand((n, SEL), device=DEV, generator=gen)
        q[get_mask_from_state(loc, SEL) != 1] = -1.0
        if level != "order":
            action = q.argmax(1)
        nxt = env.step(q.argmax(1))[0]
        bank.append_from_env(env, state, action)
        state = nxt.clone()
    env.close()
    return bank


@pytest.fixture(scope="module")
def blockout():
    from irbpp_b200 import shapes
    return shapes.make_blockout_library(32, seed=1)


@pytest.fixture(scope="module")
def location_bank(blockout):
    return filled_bank(blockout, 4096, 10, 3, "location")


@pytest.fixture(scope="module")
def order_bank(blockout):
    return filled_bank(blockout, 512, 10, 4, "order")


def nets(level, clouds, seed=7):
    torch.manual_seed(seed)
    cls, kw = (ReferenceOrderDQN, dict(buffer_size=K)) if level == "order" else (ReferenceDQN, dict(selected_action=SEL))
    online = cls(clouds, atoms=ATOMS, **kw).to(DEV).train()
    target = copy.deepcopy(online)                        # the copy shares the clouds
    target.reset_noise()
    for p in target.parameters():
        p.requires_grad = False
    return online, target


def actors(level, online, target, clouds, support):
    from irbpp_b200.actor import DeviceActor, DeviceOrderActor
    A = DeviceOrderActor if level == "order" else DeviceActor
    return A(online, clouds, support), A(target, clouds, support)


def features(level, actor, clouds, next_states, counter):
    enc = actor.effective_weights()[1] + (0.01,)
    if level == "order":
        return clouds.features(torch.arange(clouds.S, dtype=torch.int32, device=DEV), enc, counter=counter)
    return clouds.features(next_states, enc, counter=counter)


def check_target(level, bank, clouds, B):
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    online, target = nets(level, clouds)
    on_actor, tg_actor = actors(level, online, target, clouds, support)
    _, _, _, returns, next_states, nonterminals, _, _ = bank.sample(B)
    kw = "shape_features" if level == "order" else "shape_feature"
    sf_on = features(level, on_actor, clouds, next_states, 100)
    q = on_actor.q_values(next_states, **{kw: sf_on})
    a = on_actor.act(next_states, **{kw: sf_on})
    with torch.no_grad():
        q64 = (distribution(copy.deepcopy(online).double(), next_states.double(), sf_on.double()) * support.double()).sum(2)
    check_contract(q.cpu().numpy(), q64.cpu().numpy(), a.cpu().numpy(), None)      # a* within the tie tolerance
    sf_t = features(level, tg_actor, clouds, next_states, 101)
    gn = GAMMA ** N_STEP
    m, p = tg_actor.target(next_states, a, returns, nonterminals, V_MIN, V_MAX, gn, **{kw: sf_t})
    ref = target64(None, target, next_states, None, sf_t, support, returns, nonterminals, V_MIN, V_MAX, gn, next_actions=a)
    m_np, p_np = m.cpu().numpy(), p.cpu().numpy()
    dp = np.abs(p_np - ref["p"])
    assert dp.max() <= 1e-5, dp.max()
    b32 = ((torch.clamp(returns.reshape(-1, 1) + nonterminals.reshape(-1, 1) * gn * support, V_MIN, V_MAX) - V_MIN)
           / ((V_MAX - V_MIN) / (ATOMS - 1))).cpu().numpy()
    db = np.abs(b32 - ref["b"]).max(1)
    excess = np.abs(m_np - ref["m"]).sum(1) - dp.sum(1) - 2 * db
    assert excess.max() <= 1e-6, excess.max()
    m_torch = torch_projection(p, returns, nonterminals, support, V_MIN, V_MAX, gn)
    assert (m - m_torch).abs().max().item() <= 1e-6
    # a state dict gives what the live module gives
    from irbpp_b200.actor import DeviceActor, DeviceOrderActor
    A = DeviceOrderActor if level == "order" else DeviceActor
    m2, p2 = A(target.state_dict(), clouds, support, train=True).target(next_states, a, returns, nonterminals, V_MIN,
                                                                          V_MAX, gn, **{kw: sf_t})
    assert torch.equal(m, m2) and torch.equal(p, p2)
    print("%s B %d: |p - p64| %.3g, m excess %.3g, |m - m_torch| %.3g" % (
        level, B, dp.max(), excess.max(), (m - m_torch).abs().max().item()))


@pytest.mark.parametrize("B", [64, 4096])
def test_location_target_on_live_batches(blockout, location_bank, B):
    check_target("location", location_bank, clouds_for(blockout, SEL * 5), B)


@pytest.mark.parametrize("B", [64, 512])
def test_order_target_on_live_batches(blockout, order_bank, B):
    check_target("order", order_bank, clouds_for(blockout, K), B)


class _FixedBatch(object):
    """A bank that serves one recorded batch and passes priority updates on to the real bank."""

    def __init__(self, bank, batch):
        self.bank, self.batch = bank, batch

    def sample(self, batch_size):
        return self.batch

    def update_priorities(self, idxs, mem_ids, loss):
        self.bank.update_priorities(idxs, mem_ids, loss)


class _Recorder(object):
    def __init__(self, actor):
        self.actor, self.last = actor, None

    def act(self, state):
        self.last = self.actor.act(state)
        return self.last


def agent_of(online, target, B):
    return types.SimpleNamespace(online_net=online, target_net=target, batch_size=B, Vmin=V_MIN, Vmax=V_MAX,
                                 discount=GAMMA, n=N_STEP, norm_clip=10.0,
                                 optimiser=torch.optim.Adam(online.parameters(), lr=1e-4, eps=1.5e-4))


@pytest.mark.parametrize("level", ["location", "order"])
def test_device_learn_matches_the_port_learn(blockout, location_bank, order_bank, level):
    from irbpp_b200.learner_glue import device_learn
    bank = order_bank if level == "order" else location_bank
    clouds = clouds_for(blockout, K if level == "order" else SEL * 5)
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    online, target = nets(level, clouds)
    online_p, target_p = copy.deepcopy(online), copy.deepcopy(target)
    agent = agent_of(online, target, 64)
    opt_p = torch.optim.Adam(online_p.parameters(), lr=1e-4, eps=1.5e-4)
    on_actor, tg_actor = actors(level, online, target, clouds, support)
    rec = _Recorder(on_actor)
    batch = bank.sample(64)
    idxs, states, actions, returns, next_states, nonterminals, weights, mem_ids = batch
    c0 = clouds.counter
    torch.manual_seed(11)
    loss = device_learn(agent, _FixedBatch(bank, batch), rec, tg_actor)
    torch.manual_seed(11)
    target_p.reset_noise()                                 # the same draw as device_learn's
    assert all(torch.equal(a, b) for a, b in zip(target.buffers(), target_p.buffers()))
    clouds.counter = c0
    sf_states = online_p.shape_features_of(states)         # the gradient pass's index set (counter c0)
    sf_t = features(level, tg_actor, clouds, next_states, c0 + 2)
    loss_p, _ = learn_step32(online_p, target_p, opt_p, 10.0, (states, actions, returns, next_states, nonterminals,
                                                               weights), sf_states, sf_t, support, V_MIN, V_MAX,
                             GAMMA ** N_STEP, rec.last)
    dl = (loss - loss_p).abs() / (1 + loss_p.abs())
    assert dl.max().item() <= 1e-4, dl.max().item()
    worst = max(((a - b).abs().max().item() for a, b in zip(online.parameters(), online_p.parameters())))
    assert worst <= 0.05 * 1e-4, worst
    leaves = bank.tree[mem_ids.long(), idxs]
    omega = float(np.float32(bank.priority_exponent))
    assert torch.equal(leaves, (loss.detach().double() ** omega).float())      # irbpp_replay_update_kernel
    print("%s: |loss - loss_port| / (1 + |loss|) %.3g, largest parameter difference %.3g" % (level, dl.max().item(), worst))


class _SyncFreeOutsideSample(object):
    """``bank.sample`` reads its error word back (the one synchronisation it makes); everything else ``device_learn``
    does runs with torch's sync debug mode set to error."""

    def __init__(self, bank):
        self.bank = bank

    def sample(self, batch_size):
        torch.cuda.set_sync_debug_mode(0)
        try:
            return self.bank.sample(batch_size)
        finally:
            torch.cuda.set_sync_debug_mode("error")

    def update_priorities(self, idxs, mem_ids, loss):
        self.bank.update_priorities(idxs, mem_ids, loss)


def _unchecked(fn):
    def call(*a):
        torch.cuda.set_sync_debug_mode(0)
        try:
            return fn(*a)
        finally:
            torch.cuda.set_sync_debug_mode("error")
    return call


def test_hierarchical_loop_with_device_learn(blockout, location_bank, order_bank):
    """20 iterations of both learn calls (trainer.py:318-319) with update_target_net every 10, nothing but sample's
    error word leaving the device.  The target net's ``reset_noise`` (model.py:214-222, restated by the port) draws
    its noise on the host and copies it in, which torch's sync check counts; it is exempt, as sample is."""
    from irbpp_b200.learner_glue import device_learn
    support = torch.linspace(V_MIN, V_MAX, ATOMS, device=DEV)
    levels = []
    for level, bank, col in (("order", order_bank, K), ("location", location_bank, SEL * 5)):
        clouds = clouds_for(blockout, col)
        online, target = nets(level, clouds, seed=3)
        levels.append((agent_of(online, target, 64), _SyncFreeOutsideSample(bank)) + actors(level, online, target, clouds,
                                                                                            support))
    for agent, _, _, _ in levels:            # the reference's reset_noise draws on the host and copies the noise in
        agent.target_net.reset_noise = _unchecked(agent.target_net.reset_noise)
    losses = []
    try:
        torch.cuda.set_sync_debug_mode("error")
        for it in range(20):
            for agent, bank, on_actor, tg_actor in levels:
                losses.append(device_learn(agent, bank, on_actor, tg_actor))
                if (it + 1) % 10 == 0:
                    agent.target_net.load_state_dict(agent.online_net.state_dict())     # Agent.update_target_net
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(bool(torch.isfinite(l).all()) for l in losses)


@pytest.mark.parametrize("case", ["loc_default", "loc_exact", "order_default", "order_exact"])
def test_reference_fixture_through_the_target_actors(case):
    """``learn.npz`` (the unmodified reference's ``Agent.learn``): with the fixture's online net and the target noise
    ``learn`` drew, the device actors' a* and ``m`` give the reference's loss within ``1e-4 (1 + |loss|)``, from the
    live target module and from its state dict."""
    from irbpp_b200.actor import DeviceActor, DeviceOrderActor
    from test_learn_golden import case_inputs, constants, shape_features
    from conftest import load_golden
    from test_actor import decode_fixture
    from test_order_actor import decode_fixture as decode_order_fixture
    gx = dict(learn=dict(load_golden("learn")), loc=decode_fixture(load_golden("dqn_act")),
              order=decode_order_fixture(load_golden("dqn_order_act")))
    gn = constants(gx)[0]
    level, online, target, b, support, v_min, v_max, points = case_inputs(gx, case, DEV)
    A, kw = (DeviceOrderActor, "shape_features") if level == "order" else (DeviceActor, "shape_feature")
    with torch.no_grad():
        sf_on = shape_features(level, online, points, b["next_states"])
        sf_t = shape_features(level, target, points, b["next_states"])
        log_ps_a = distribution(online, b["states"], shape_features(level, online, points, b["states"]), log=True)[
            torch.arange(b["states"].shape[0], device=DEV), b["actions"]]
    a = A(online, None, support).act(b["next_states"], **{kw: sf_on})
    want = gx["learn"][case + ":loss"]
    for tg in (A(target, None, support), A(target.state_dict(), None, support, train=True)):
        m, p = tg.target(b["next_states"], a, b["returns"], b["nonterminals"], v_min, v_max, gn, **{kw: sf_t})
        loss = -(m * log_ps_a).sum(1).cpu().numpy()
        err = np.abs(loss - want) / (1 + np.abs(want))
        assert err.max() <= 1e-4, err.max()
    print("%s: |loss - reference| / (1 + |loss|) %.3g" % (case, err.max()))
