"""``DeviceActor`` (``csrc/irbpp_actor.cuh``) on the GPU against ``oracle/dqn_port.py`` run in float64 on the device.

Accuracy contract (as in tests/test_actor.py): ``|q - q64| <= 1e-4 * (1 + |q64|)`` on every row; the action equals
``argmax q64`` unless the float64 top-two gap among the unmasked rows is below ``2e-4 * (1 + |max|)``, where any row
within that gap is taken; a fully masked bin acts 0."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.dqn_port import DQNPort
from test_actor import SEL, check_contract, decode_fixture, port_from

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def fx():
    return decode_fixture(load_golden("dqn_act"))


def port64_q(net, obs, sf, support, chunk=256):
    """Unmasked expected values of the float64 port on the device, in chunks of bins (intermediates of
    [bins * sel, 512] float64)."""
    net64 = DQNPort(selected_action=net.sel, atoms=net.atoms).to(DEV, torch.float64)
    net64.load_state_dict({k: v.to(DEV, torch.float64) for k, v in net.state_dict().items()})
    net64.train(net.training)
    out = []
    with torch.no_grad():
        for i in range(0, obs.shape[0], chunk):
            out.append(net64.sum_q(obs[i:i + chunk].double(), sf[i:i + chunk].double(), support.double()))
    return torch.cat(out).cpu().numpy()


def contract(actor, net, obs, sf, support, label):
    from irbpp_b200.learner_glue import get_mask_from_state
    sel = net.sel
    mask = get_mask_from_state(obs, sel)
    q64 = port64_q(net, obs, sf, support)
    m = mask.cpu().numpy()
    q = actor.q_values(obs, mask, shape_feature=sf).cpu().numpy()
    act = actor.act(obs, mask, shape_feature=sf).cpu().numpy()
    worst = check_contract(q, np.where(m == 1, q64, -np.inf), act, m)
    qu = actor.q_values(obs, shape_feature=sf).cpu().numpy()
    worst = max(worst, check_contract(qu, q64, actor.act(obs, shape_feature=sf).cpu().numpy(), None))
    print("%s: largest |q - q64| / (1 + |q64|) = %.3g over %d bins" % (label, worst, obs.shape[0]))
    return act


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_fixture_through_device_actor(fx, mode):
    from irbpp_b200.actor import DeviceActor
    from test_actor import shape_features
    net = port_from(fx, mode == "train", torch.float32).to(DEV)
    sd = {k[3:]: torch.tensor(v) for k, v in fx.items() if k.startswith("sd:")}
    support = torch.tensor(fx["support"], device=DEV)
    obs = torch.tensor(fx["obs"], device=DEV)
    sf = shape_features(fx, port_from(fx, True, torch.float32)).to(DEV)
    act_sd = contract(DeviceActor(sd, None, support, train=(mode == "train")), net, obs, sf, support, "fixture " + mode)
    act_live = DeviceActor(net, None, support).act(obs, obs[:, :SEL * 5].reshape(-1, SEL, 5)[:, :, 4], shape_feature=sf)
    assert np.array_equal(act_sd, act_live.cpu().numpy())


def live_bins(lib, n, steps, seed):
    from irbpp_b200.learner_glue import get_mask_from_state
    from irbpp_b200.vec_env import GpuVecEnv
    env = GpuVecEnv(lib, None, num_envs=n, device=DEV, item_seed=seed)
    state = env.reset()
    gen = torch.Generator(device=DEV); gen.manual_seed(seed)
    for _ in range(steps):                   # burn-in with random valid actions
        q = torch.rand((n, SEL), device=DEV, generator=gen)
        q[get_mask_from_state(state, SEL) != 1] = -1.0
        state = env.step(q.argmax(1))[0]
    state = state.clone()
    env.close()
    return state


@pytest.mark.parametrize("workload", ["blockout", "irregular8"])
def test_live_bins_4096(workload):
    from irbpp_b200 import shapes
    from irbpp_b200.actor import DeviceActor
    from irbpp_b200.pointnet import DeviceShapeClouds
    torch.manual_seed(1)
    lib = shapes.make_blockout_library(32, seed=1) if workload == "blockout" else shapes.make_irregular_library(16, seed=2, num_rotations=8)
    state = live_bins(lib, 4096, 12, 3)
    net = DQNPort().to(DEV).train()
    support = torch.linspace(-10, 10, 31, device=DEV)
    clouds = DeviceShapeClouds(np.random.default_rng(0).random((lib.num_shapes, 4096, 3)).astype(np.float32) * 0.1, device=DEV)
    actor = DeviceActor(net, clouds, support)
    from irbpp_b200.learner_glue import get_mask_from_state
    a_clouds = actor.act(state, get_mask_from_state(state, SEL))
    sf = clouds.features(state, actor.effective_weights()[1] + (0.01,), counter=clouds.counter - 1)
    act = contract(actor, net, state, sf, support, "4096 live %s bins" % workload)
    assert np.array_equal(a_clouds.cpu().numpy(), act)


def test_weights_followed_after_learning_step(fx):
    """An optimiser step and reset_noise() change the weights; the next act follows them (nothing is cached)."""
    from irbpp_b200.actor import DeviceActor
    from test_actor import shape_features
    net = port_from(fx, True, torch.float32).to(DEV)
    support = torch.tensor(fx["support"], device=DEV)
    obs = torch.tensor(fx["obs"], device=DEV)
    sf = shape_features(fx, port_from(fx, True, torch.float32)).to(DEV)
    actor = DeviceActor(net, None, support)
    q_before = actor.q_values(obs, shape_feature=sf).clone()
    opt = torch.optim.Adam(net.parameters(), lr=1e-2)
    loss = -(net(obs, sf) * support).sum(2).mean()
    opt.zero_grad(); loss.backward(); opt.step()
    net.reset_noise()
    q_after = actor.q_values(obs, shape_feature=sf)
    assert not torch.equal(q_before, q_after)
    contract(actor, net, obs, sf, support, "after a learning step")


def test_saved_state_dict_matches_live_module(fx, tmp_path):
    from irbpp_b200.actor import DeviceActor
    from test_actor import shape_features
    net = port_from(fx, True, torch.float32).to(DEV)
    path = str(tmp_path / "model.pt")
    torch.save(net.state_dict(), path)
    support = torch.tensor(fx["support"], device=DEV)
    obs = torch.tensor(fx["obs"], device=DEV)
    sf = shape_features(fx, port_from(fx, True, torch.float32)).to(DEV)
    mask = obs[:, :SEL * 5].reshape(-1, SEL, 5)[:, :, 4]
    live = DeviceActor(net, None, support).act(obs, mask, shape_feature=sf)
    saved = DeviceActor(torch.load(path, map_location="cpu"), None, support, train=True).act(obs, mask, shape_feature=sf)
    assert torch.equal(live, saved)


def test_argument_errors(fx):
    from irbpp_b200.actor import DeviceActor
    sd = {k[3:]: torch.tensor(v) for k, v in fx.items() if k.startswith("sd:")}
    actor = DeviceActor(sd, None, torch.tensor(fx["support"], device=DEV))
    obs = torch.tensor(fx["obs"], device=DEV)
    sf = torch.zeros((obs.shape[0], 128), device=DEV)
    with pytest.raises(ValueError, match="CUDA"):
        actor.act(obs.cpu(), shape_feature=sf)
    with pytest.raises(ValueError, match="observation width"):
        actor.act(obs[:, 1:], shape_feature=sf[:, :])
    with pytest.raises(ValueError, match="shape_feature"):
        actor.act(obs, shape_feature=sf[:3])
    with pytest.raises(ValueError, match="no DeviceShapeClouds"):
        actor.act(obs)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="lives on"):
            actor.act(obs.to("cuda:1"), shape_feature=sf)


def test_evaluate_with_idle_bins(fx):
    """evaluate(policy=actor.act) over 6 trajectories on 8 bins (two idle from the start, more as trajectories end)."""
    from irbpp_b200 import shapes
    from irbpp_b200.actor import DeviceActor
    from irbpp_b200.evaluation import evaluate
    from irbpp_b200.learner_glue import get_mask_from_state
    from irbpp_b200.pointnet import DeviceShapeClouds
    lib = shapes.make_blockout_library(8, seed=1)
    rng = np.random.default_rng(4)
    trajs = [list(rng.integers(0, lib.num_shapes, 300)) for _ in range(6)]
    sd = {k[3:]: torch.tensor(v) for k, v in fx.items() if k.startswith("sd:")}
    clouds = DeviceShapeClouds(fx["shape_array"], device=DEV)
    actor = DeviceActor(sd, clouds, torch.tensor(fx["support"], device=DEV), train=False)
    res = evaluate(lib, trajs, lambda obs: actor.act(obs, get_mask_from_state(obs, SEL)), num_envs=8, first=0, count=6)
    assert len(res["trajectory"]) == 6 and (res["length"] > 0).all() and (res["ratio"] > 0).all()


def test_fine_action_grid():
    """The 32 x 32 action grid (resolutionA = 0.01): the network does not depend on the grid."""
    from irbpp_b200 import shapes
    from irbpp_b200.actor import DeviceActor
    from irbpp_b200.learner_glue import get_mask_from_state
    from irbpp_b200.vec_env import GpuVecEnv
    torch.manual_seed(2)
    lib = shapes.make_blockout_library(12, seed=4, resolutionAct=0.01)
    env = GpuVecEnv(lib, None, num_envs=256, device=DEV, item_seed=5)
    state = env.reset()
    net = DQNPort().to(DEV).train()
    support = torch.linspace(-10, 10, 31, device=DEV)
    actor = DeviceActor(net, None, support)
    sf = torch.randn((256, 128), device=DEV) * 0.1
    for _ in range(4):
        state = env.step(actor.act(state, get_mask_from_state(state, SEL), shape_feature=sf))[0]
    state = state.clone()
    env.close()
    contract(actor, net, state, sf, support, "fine grid")
