"""``DeviceOrderActor`` (``csrc/irbpp_order_actor.cuh``) on the GPU against ``oracle/order_dqn_port.py`` run in float64
on the device, and the hierarchical actor loop (order act, candidates, location act, step) on the device.

Accuracy contract (as in tests/test_actor.py, over the k slots): ``|q - q64| <= 1e-4 * (1 + |q64|)``; the action
equals ``argmax q64`` unless the float64 top-two gap among the unmasked slots is below ``2e-4 * (1 + |max|)``; a fully
masked bin acts 0."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.order_dqn_port import OrderDQNPort
from test_actor import check_contract
from test_actor_range import support_for
from test_order_actor import (ATOMS, KS, decode_fixture, fixture_sd, make_obs, order_act, port_from, seeded_net,
                              shape_table)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = torch.device("cuda:0")
SEL = 500


@pytest.fixture(scope="module")
def fx():
    return decode_fixture(load_golden("dqn_order_act"))


def port64_q(net, obs, sf, support, mask=None, chunk=1024):
    """Expected values of the float64 port on the device (-inf where mask != 1)."""
    net64 = OrderDQNPort(buffer_size=net.k, atoms=net.atoms).to(DEV, torch.float64)
    net64.load_state_dict({k: v.to(DEV, torch.float64) for k, v in net.state_dict().items()})
    net64.train(net.training)
    out = []
    with torch.no_grad():
        for i in range(0, obs.shape[0], chunk):
            out.append(net64.sum_q(obs[i:i + chunk].to(DEV).double(), sf.to(DEV).double(), support.to(DEV).double(),
                                   None if mask is None else mask[i:i + chunk].to(DEV)))
    return torch.cat(out).cpu().numpy()


def contract(actor, net, obs, sf, support, label, mask=None):
    q64 = port64_q(net, obs, sf, support, mask)
    q = actor.q_values(obs, mask, shape_features=sf).cpu().numpy()
    act = actor.act(obs, mask, shape_features=sf).cpu().numpy()
    worst = check_contract(q, q64, act, None if mask is None else mask.cpu().numpy())
    print("%s: largest |q - q64| / (1 + |q64|) = %.3g over %d bins" % (label, worst, obs.shape[0]))
    return act, worst


def clouds_for(lib, points=4096, seed=0):
    from irbpp_b200.pointnet import DeviceShapeClouds
    arr = np.random.default_rng(seed).random((lib.num_shapes, points, 3)).astype(np.float32) * 0.1
    return DeviceShapeClouds(arr, device=DEV, item_col=SEL * 5)


def order_states(lib, n, k, steps, seed):
    """Order observations of n live bins after ``steps`` hierarchical steps with random slots and random valid
    candidates."""
    from irbpp_b200.learner_glue import get_mask_from_state
    from irbpp_b200.vec_env import GpuVecEnv
    env = GpuVecEnv(lib, None, num_envs=n, device=DEV, buffer_size=k, item_seed=seed)
    state = env.reset()
    gen = torch.Generator(device=DEV); gen.manual_seed(seed)
    for _ in range(steps):
        order = torch.randint(0, k, (n,), device=DEV, generator=gen)
        loc = env.get_action_candidates(order, as_tensor=True)
        q = torch.rand((n, SEL), device=DEV, generator=gen)
        q[get_mask_from_state(loc, SEL) != 1] = -1.0
        state = env.step(q.argmax(1))[0]
    state = state.clone()
    env.close()
    return state


@pytest.mark.parametrize("workload", ["blockout", "irregular8"])
def test_live_bins_4096(workload):
    from irbpp_b200 import shapes
    from irbpp_b200.actor import DeviceOrderActor
    torch.manual_seed(1)
    lib = shapes.make_blockout_library(32, seed=1) if workload == "blockout" else shapes.make_irregular_library(16, seed=2, num_rotations=8)
    state = order_states(lib, 4096, 10, 12, 3)
    assert state.shape == (4096, 10 + 1024) and (state[:, 10:] > 0).any()
    net = OrderDQNPort(buffer_size=10).to(DEV).train()
    support = torch.linspace(-10, 10, 31, device=DEV)
    clouds = clouds_for(lib)
    actor = DeviceOrderActor(net, clouds, support)
    a_clouds = actor.act(state)
    ids = torch.arange(lib.num_shapes, dtype=torch.int32, device=DEV)
    sf = clouds.features(ids, actor.effective_weights()[1] + (0.01,), counter=clouds.counter - 1)
    act, _ = contract(actor, net, state, sf, support, "4096 live %s bins, k 10" % workload)
    assert np.array_equal(a_clouds.cpu().numpy(), act)


@pytest.mark.parametrize("k", KS)
def test_full_range_1024(fx, k):
    """Every atom count at every k, 1024 bins each, from a state dict in its mode; masked and unmasked."""
    from irbpp_b200.actor import DeviceOrderActor
    for i, atoms in enumerate(ATOMS):
        mode = ("train", "eval", "reset_noise")[(i + k) % 3]
        net = seeded_net(k, atoms, mode).to(DEV)
        support = torch.tensor(support_for(atoms), device=DEV)
        obs = torch.tensor(make_obs(fx, k, 1024, 8, seed=k + atoms), device=DEV)
        sf = shape_table(net, fx["clouds"])
        actor = DeviceOrderActor({n: v.cpu() for n, v in net.state_dict().items()}, None, support, train=net.training)
        mask = (torch.rand((1024, k), device=DEV) < 0.7).float()
        mask[:3] = 0.0
        contract(actor, net, obs, sf, support, "k %d, atoms %d, %s" % (k, atoms, mode))
        contract(actor, net, obs, sf, support, "k %d, atoms %d, %s, masked" % (k, atoms, mode), mask)


def test_live_module_follows_reset_noise_and_learning(fx):
    from irbpp_b200.actor import DeviceOrderActor
    net = port_from(fx, 10, True, torch.float32).to(DEV)
    support = torch.tensor(fx["support"], device=DEV)
    obs = torch.tensor(fx["obs10"], device=DEV)
    sf = shape_table(net, fx["clouds"])
    actor = DeviceOrderActor(net, None, support)
    q0 = actor.q_values(obs, shape_features=sf).clone()
    net.reset_noise()
    q1 = actor.q_values(obs, shape_features=sf).clone()
    assert not torch.equal(q0, q1)
    contract(actor, net, obs, sf, support, "after reset_noise")
    opt = torch.optim.Adam(net.parameters(), lr=1e-2)
    loss = -(net(obs, sf) * support).sum(2).mean()
    opt.zero_grad(); loss.backward(); opt.step()
    assert not torch.equal(q1, actor.q_values(obs, shape_features=sf))
    contract(actor, net, obs, sf, support, "after a learning step")
    net.eval()
    contract(actor, net, obs, sf, support, "eval mode")


def test_fixture_through_device_actor(fx):
    """The reference's recorded actions, through a saved state dict."""
    from irbpp_b200.actor import DeviceOrderActor
    support = torch.tensor(fx["support"], device=DEV)
    for k in (3, 10):
        for mode in ("train", "eval"):
            net = port_from(fx, k, mode == "train", torch.float32).to(DEV)
            sf = shape_table(net, fx["clouds"])
            obs = torch.tensor(fx["obs%d" % k], device=DEV)
            act, _ = contract(DeviceOrderActor(fixture_sd(fx), None, support, train=(mode == "train")), net, obs, sf,
                              support, "fixture k %d %s" % (k, mode))
            assert np.array_equal(act, fx["%s_action%d" % (mode, k)])


def test_raw_entry_wide_stride_and_separate_mask(fx):
    from irbpp_b200 import _lib
    lib = _lib.load()
    k = 10
    net = seeded_net(k, 31, "train").to(DEV)
    obs = torch.tensor(make_obs(fx, k, 1024, 8, seed=9), device=DEV)
    wide = torch.full((1024, obs.shape[1] + 40), float("nan"), device=DEV)
    wide[:, 7:7 + obs.shape[1]] = obs
    view = wide[:, 7:7 + obs.shape[1]]
    sf = shape_table(net, fx["clouds"])
    support = torch.tensor(support_for(31), device=DEV)
    store = torch.zeros((1024, 2 * k), device=DEV)
    store[:, ::2] = (torch.rand((1024, k), device=DEV) < 0.5).float()
    mask = store[:, ::2]                                  # element stride 2
    q64 = port64_q(net, obs, sf, support, mask)
    act, q = order_act(lib, net, view, k, sf, support, mask, prefix="")
    worst = check_contract(q, q64, act, mask.cpu().numpy())
    act_only, none = order_act(lib, net, view, k, sf, support, mask, want_q=False, prefix="")
    assert none is None and np.array_equal(act_only, act)
    print("raw entry, obs_stride %d, mask element stride 2: largest scaled error %.3g" % (wide.shape[1], worst))


def test_order_point_rule_on_device():
    """OrderShapeClouds' features equal the shape encoder on the points order_point_indices names, across a redraw."""
    from irbpp_b200 import shapes
    from irbpp_b200.pointnet import OrderShapeClouds, order_point_indices
    lib = shapes.make_blockout_library(8, seed=1)
    clouds = clouds_for(lib, points=12000, seed=4)
    rule = OrderShapeClouds(clouds)
    net = OrderDQNPort().to(DEV)
    ids = torch.arange(lib.num_shapes, dtype=torch.int32, device=DEV)
    enc = tuple(p.detach() for p in (net.shapeEncoder.linear1.weight, net.shapeEncoder.linear1.bias,
                                     net.shapeEncoder.linear2.weight, net.shapeEncoder.linear2.bias)) + (0.01,)
    for c in (0, 999, 1000, 2345):
        got = rule.features(ids, enc, counter=c)
        idx = torch.as_tensor(order_point_indices(clouds.seed, c, 1024, clouds.P), device=DEV)
        with torch.no_grad():
            want = net.shape_feature(clouds.shape_array[:, idx])
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
    assert rule.counter == 0
    rule.features(ids, enc)
    assert rule.counter == 1


def test_hierarchical_loop_on_device(fx):
    """trainer_hierarchical's three calls, 30 iterations at 1024 bins, nothing leaving the device: order act,
    get_action_candidates(as_tensor=True), location act, step.  The order actions of the last iteration meet the
    contract."""
    from irbpp_b200 import shapes
    from irbpp_b200.actor import DeviceActor, DeviceOrderActor
    from irbpp_b200.learner_glue import get_mask_from_state
    from irbpp_b200.pointnet import OrderShapeClouds
    from irbpp_b200.vec_env import GpuVecEnv
    from oracle.dqn_port import DQNPort
    torch.manual_seed(3)
    lib = shapes.make_blockout_library(32, seed=1)
    clouds = clouds_for(lib, points=10000)
    order_net = OrderDQNPort(buffer_size=10).to(DEV).train()
    loc_net = DQNPort().to(DEV).train()
    support = torch.linspace(-10, 10, 31, device=DEV)
    order_actor = DeviceOrderActor(order_net, OrderShapeClouds(clouds), support)
    loc_actor = DeviceActor(loc_net, clouds, support)
    env = GpuVecEnv(lib, None, num_envs=1024, device=DEV, buffer_size=10, item_seed=7)
    state = env.reset()
    placed = 0.0
    for _ in range(30):
        order = order_actor.act(state)
        loc = env.get_action_candidates(order, as_tensor=True)
        action = loc_actor.act(loc, get_mask_from_state(loc, SEL))
        last = state
        state, reward, done, _ = env.step(action)
        placed += float(reward.sum())
    env.close()
    assert placed > 0
    ids = torch.arange(lib.num_shapes, dtype=torch.int32, device=DEV)
    sf = order_actor.clouds.features(ids, order_actor.effective_weights()[1] + (0.01,), counter=29)
    act, _ = contract(order_actor, order_net, last, sf, support, "hierarchical loop, last iteration")
    assert np.array_equal(act, order.cpu().numpy())


def test_evaluate_buffered_with_both_device_actors(fx):
    """evaluate(..., buffer_size=10, order_policy=...) over 6 trajectories on 8 bins; every order action equals the
    float64 port's wherever the port's top-two margin exceeds the contract."""
    from irbpp_b200 import shapes
    from irbpp_b200.actor import DeviceActor, DeviceOrderActor
    from irbpp_b200.evaluation import evaluate
    from irbpp_b200.learner_glue import get_mask_from_state
    from oracle.dqn_port import DQNPort
    torch.manual_seed(4)
    lib = shapes.make_blockout_library(8, seed=1)
    rng = np.random.default_rng(4)
    trajs = [list(rng.integers(0, lib.num_shapes, 200)) for _ in range(6)]
    clouds = clouds_for(lib)
    support = torch.linspace(-10, 10, 31, device=DEV)
    order_net = OrderDQNPort(buffer_size=10).to(DEV).eval()
    order_actor = DeviceOrderActor(order_net, clouds, support)
    loc_actor = DeviceActor(DQNPort().to(DEV).eval(), clouds, support)
    ids = torch.arange(lib.num_shapes, dtype=torch.int32, device=DEV)
    seen = []

    def order_policy(obs):
        sf = clouds.features(ids, order_actor.effective_weights()[1] + (0.01,))
        a = order_actor.act(obs, shape_features=sf)
        seen.append((obs.clone(), sf, a.clone()))
        return a

    res = evaluate(lib, trajs, lambda obs: loc_actor.act(obs, get_mask_from_state(obs, SEL)), num_envs=8, first=0,
                   count=6, order_policy=order_policy, buffer_size=10)
    assert len(res["trajectory"]) == 6 and (res["length"] > 0).all() and (res["ratio"] > 0).all()
    obs = torch.cat([o for o, _, _ in seen])
    act = torch.cat([a for _, _, a in seen]).cpu().numpy()
    q64 = np.concatenate([port64_q(order_net, o, sf, support) for o, sf, _ in seen])
    check_contract(q64.astype(np.float32), q64, act, None)
    print("evaluate, buffer 10: %d order acts, %d bins each" % (len(seen), obs.shape[0] // len(seen)))
