"""Generate ``learn.npz`` from the UNMODIFIED reference ``Agent`` (``agent.py``) and network (``model.py`` ``DQNBPP``).

Run in the build container (needs the reference tree and torch):

    python tests/golden/make_golden_learn.py

``model.py`` and ``agent.py`` are executed from where they lie, after ``oracle/ref_loader.py`` has installed its import
stand-ins (``agent.py`` imports ``DQNBPP`` from ``model``).  An ``Agent`` is built on the CPU from a ``SimpleNamespace``
of arguments, for both network levels:

* location: ``selectedAction = 500``, the network of ``dqn_act.npz`` (its quantised weights and compact noise), next
  states from that fixture's observations (live BlockOut bins, truncated irregular bins, single-row bins and blank
  all-zero bins, as ``memory.py:106,147`` produces them);
* order: ``bufferSize = k = 10``, the network of ``dqn_order_act.npz``, states from its ``obs10`` (the last two rows
  blank).

The online net gets the fixture's state dict, ``update_target_net`` copies it to the target net.  Every point of a
shape's cloud is the same (the fixture cloud's first point), so the shape feature does not depend on the point indices
the reference draws with ``np.random`` and the fixture does not depend on point RNG.

Each level is run on two supports (31 atoms, the fixtures' networks): the reference defaults ``V_min = -1``,
``V_max = 8``, and an exact grid ``-15 .. 15`` (dz = 1) whose returns hit the edge cases exactly: ``b`` an integer in
the interior, at 0 and at ``atoms - 1``, ``Tz`` clamped at both ends, ``nonterminal = 0``, blank next states.

``Agent.learn`` draws the batch from two stub memories (``segment_size = 4``) that return fixed ``(idx, state, action,
R, next_state, nonterminal, weight)`` and record what ``update_priorities`` receives.  Recorded per case (``<case>`` is
``loc_default``, ``loc_exact``, ``order_default``, ``order_exact``):

* ``<case>:state_rows`` / ``next_rows`` (rows of the source fixture's observations), ``actions``, ``returns``,
  ``nonterminals``, ``weights``, ``v_min``, ``v_max``;
* ``<case>:loss`` (what ``learn`` returns) and ``<case>:priorities`` (what it passes to ``update_priorities``);
* the target net's noise after ``learn``'s ``target_net.reset_noise()`` by its factors, ``<case>:tnoise_in:<layer>``
  and ``<case>:tnoise_out:<layer>`` (``weight_epsilon`` is their float32 outer product, checked bit for bit here);
* the online parameters after the Adam step: per parameter 32 flat positions (``<case>:pidx:<key>``, seeded) and
  their values (``<case>:pval:<key>``), and the float64 sum of the whole tensor (``<case>:psum:<key>``).

``learn.npz`` as committed was written by this script with numpy 2.3.5 and torch 2.11.
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_loader  # noqa: E402

SEL, K, ATOMS = 500, 10, 31
BATCH, MEMORIES = 8, 2
GAMMA, N_STEP, NORM_CLIP, LR, ADAM_EPS = 0.99, 3, 10.0, 6.25e-5, 1.5e-4
SUPPORTS = {"default": (-1.0, 8.0), "exact": (-15.0, 15.0)}
NOISY = ("fc_h_v", "fc_h_a", "fc_z_v", "fc_z_a")           # DQNBPP.reset_noise's order (named_children)
SAMPLES = 32


def load_reference_modules():
    ref_loader.load_reference()
    mods = {}
    for name in ("model", "agent"):
        spec = importlib.util.spec_from_file_location(name, os.path.join(ref_loader.REFERENCE_ROOT, name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod               # agent.py: from model import DQNBPP
        spec.loader.exec_module(mod)
        mods[name] = mod
    return mods["model"], mods["agent"]


class StubMemory(object):
    """``ReplayMemory.sample`` / ``update_priorities`` with fixed transitions."""

    def __init__(self, idx, state, action, R, next_state, nonterminal, weight):
        self.out = (idx, state, action, R, next_state, nonterminal, weight)
        self.priorities = None

    def sample(self, segment):
        assert segment == self.out[1].shape[0]
        return self.out

    def update_priorities(self, idx, priorities):
        self.priorities = priorities.numpy().copy()


def batch(case, level, n_rows, blank_rows):
    """Rows, actions, returns, nonterminals, weights of one case (seeded)."""
    rng = np.random.default_rng(sum(map(ord, case)))
    live = [r for r in range(n_rows) if r not in blank_rows]
    state_rows = rng.choice(live, BATCH)
    next_rows = rng.choice(live, BATCH)
    next_rows[[2, 6]] = blank_rows[:2]                      # blank next states (memory.py:106,147)
    actions = rng.integers(0, SEL if level == "loc" else K, BATCH)
    weights = rng.uniform(0.3, 1.0, BATCH).astype(np.float32)
    weights[weights.argmax()] = 1.0
    if case.endswith("exact"):
        # b = 18 (interior), b = 0, b = 30, Tz clamped below and above, b = 17.5, then two nonterminal draws
        returns = np.array([3.0, -15.0, 15.0, -40.0, 40.0, 2.5, 0.25, -6.0], np.float32)
        nonterminals = np.array([0, 0, 0, 1, 1, 0, 1, 1], np.float32)
    else:
        returns = rng.uniform(-3.0, 12.0, BATCH).astype(np.float32)
        nonterminals = (rng.random(BATCH) < 0.7).astype(np.float32)
        nonterminals[0] = 0.0
    return state_rows, next_rows, actions, returns, nonterminals, weights


def run_case(model, agent_mod, case, level, sd, obs, constant_points, blank_rows, out):
    import torch
    v_min, v_max = SUPPORTS[case.split("_")[1]]
    S = constant_points.shape[0]
    npts = 10000 if level == "order" else 2048              # the order level subsamples 10 000 points (model.py:240-244)
    shape_array = np.repeat(constant_points[:, None, :], npts, axis=1)
    args = types.SimpleNamespace(
        action_space=SEL if level == "loc" else K, atoms=ATOMS, V_min=v_min, V_max=v_max, device=torch.device("cpu"),
        batch_size=BATCH, multi_step=N_STEP, discount=GAMMA, norm_clip=NORM_CLIP, shapeArray=shape_array, model="",
        learning_rate=LR, adam_eps=ADAM_EPS, selectedAction=SEL, level="order" if level == "order" else "location",
        heightMap=True, ZRotNum=4, bin_dimension=[0.32, 0.32, 0.30], resolutionH=0.01,
        bufferSize=K if level == "order" else 1, hidden_size=128, noisy_std=0.5, samplePointsNum=1024)
    torch.manual_seed(1)
    np.random.seed(1)
    agent = agent_mod.Agent(args)
    agent.online_net.load_state_dict({k: torch.tensor(v) for k, v in sd.items()})
    agent.update_target_net()
    state_rows, next_rows, actions, returns, nonterminals, weights = batch(case, level, obs.shape[0], blank_rows)
    seg = BATCH // MEMORIES
    mems = []
    for i in range(MEMORIES):
        s = slice(i * seg, (i + 1) * seg)
        mems.append(StubMemory(np.arange(seg) + 100 * i, torch.tensor(obs[state_rows[s]]), torch.tensor(actions[s]),
                               torch.tensor(returns[s]), torch.tensor(obs[next_rows[s]]),
                               torch.tensor(nonterminals[s]), torch.tensor(weights[s])))
    rng_state = torch.get_rng_state()
    loss = agent.learn(mems)                                 # agent.py:68-125, unmodified
    torch.set_rng_state(rng_state)                           # replay learn's only torch draws: target_net.reset_noise()
    f = lambda n: (lambda x: x.sign().mul_(x.abs().sqrt_()))(torch.randn(n))
    for name in NOISY:
        mod = getattr(agent.target_net, name)
        e_in, e_out = f(mod.in_features), f(mod.out_features)
        assert np.array_equal(np.outer(e_out.numpy(), e_in.numpy()), mod.weight_epsilon.numpy()), name
        assert np.array_equal(e_out.numpy(), mod.bias_epsilon.numpy()), name
        out["%s:tnoise_in:%s" % (case, name)], out["%s:tnoise_out:%s" % (case, name)] = e_in.numpy(), e_out.numpy()
    prng = np.random.default_rng(77)
    for key, p in agent.online_net.named_parameters():
        v = p.detach().numpy().reshape(-1)
        idx = prng.choice(v.size, min(SAMPLES, v.size), replace=False).astype(np.int32)
        out["%s:pidx:%s" % (case, key)], out["%s:pval:%s" % (case, key)] = idx, v[idx]
        out["%s:psum:%s" % (case, key)] = np.float64(v.astype(np.float64).sum())
    out.update({"%s:%s" % (case, k): v for k, v in dict(
        state_rows=state_rows.astype(np.int32), next_rows=next_rows.astype(np.int32), actions=actions.astype(np.int64),
        returns=returns, nonterminals=nonterminals, weights=weights, v_min=np.float64(v_min), v_max=np.float64(v_max),
        loss=loss.detach().numpy(), priorities=np.concatenate([m.priorities for m in mems])).items()})
    print(case, "loss", np.round(loss.detach().numpy(), 4))


def main():
    from conftest import load_golden
    from test_actor import decode_fixture
    from test_order_actor import decode_fixture as decode_order_fixture
    model, agent_mod = load_reference_modules()
    out = {"batch": np.int32(BATCH), "memories": np.int32(MEMORIES), "discount": np.float64(GAMMA),
           "multi_step": np.int32(N_STEP), "norm_clip": np.float64(NORM_CLIP), "learning_rate": np.float64(LR),
           "adam_eps": np.float64(ADAM_EPS)}
    fx = decode_fixture(load_golden("dqn_act"))
    sd = {k[3:]: v for k, v in fx.items() if k.startswith("sd:")}
    blank = [int(r) for r in np.nonzero(fx["kinds"] == 4)[0]]
    for case in ("loc_default", "loc_exact"):
        run_case(model, agent_mod, case, "loc", sd, fx["obs"], fx["shape_array"][:, 0], blank, out)
    ofx = decode_order_fixture(load_golden("dqn_order_act"))
    osd = {k[3:]: v for k, v in ofx.items() if k.startswith("sd:")}
    obs10 = ofx["obs10"]
    for case in ("order_default", "order_exact"):
        run_case(model, agent_mod, case, "order", osd, obs10, ofx["clouds"][:, 0], [obs10.shape[0] - 2, obs10.shape[0] - 1],
                 out)
    path = os.path.join(HERE, "learn.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
