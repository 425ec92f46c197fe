"""The prioritized n-step replay on the H100 (``pytest -m gpu``): the fixture of the unmodified ``memory.py`` replayed
through ``learner_glue.PrioritizedReplayBank``; 4096 memories fed by a real ``GpuVecEnv`` against
``oracle/replay_port.py`` on the same data and uniforms; the order-level observation width; the bounded draws."""
import numpy as np
import pytest

import replay_checks as rc

pytestmark = pytest.mark.gpu


def _dev():
    import torch
    return torch.device("cuda:0")


class BankBackend(object):
    """``PrioritizedReplayBank`` behind the fixture driver's backend interface."""

    def __init__(self, M, C, L, discount, n, beta, omega):
        from irbpp_b200.learner_glue import PrioritizedReplayBank
        self.bank = PrioritizedReplayBank(M, C, L, _dev(), discount, n, beta, omega, seed=5)

    def append(self, state, action, reward, done, valid, clip):
        import torch
        self.bank.append_batch(torch.from_numpy(np.ascontiguousarray(state)).to(_dev()), action, reward, done, valid,
                               reward_clip=clip)

    def sample(self, mem_ids, k, uniforms, beta):
        import torch
        self.bank.priority_weight = beta
        ids = torch.from_numpy(np.ascontiguousarray(mem_ids, np.int32)).to(_dev())
        U = torch.from_numpy(np.ascontiguousarray(uniforms)).to(_dev()) if uniforms is not None else None
        res = self.bank._sample(ids, k, U)
        names = ("tree_idx", "states", "actions", "returns", "next_states", "nonterminals", "weights")
        out = {n: res[i].cpu().numpy().reshape(-1) if n != "states" and n != "next_states" else res[i].cpu().numpy()
               for i, n in enumerate(names)}
        out["attempts"] = self.bank.last_attempts.cpu().numpy()
        out["error"] = self.bank.last_error.cpu().numpy()
        return out

    def update(self, mem_ids, tree_idxs, loss):
        import torch
        self.bank.update_priorities(torch.from_numpy(np.asarray(tree_idxs, np.int64)).to(_dev()),
                                    torch.from_numpy(np.asarray(mem_ids, np.int32)).to(_dev()),
                                    torch.from_numpy(np.asarray(loss, np.float32)).to(_dev()))

    def snapshot(self):
        st = self.bank.state.cpu().numpy()
        return (self.bank.tree.cpu().numpy(), st[:, 0].copy(), st[:, 1].copy(), st[:, 2].copy(),
                st[:, 3].copy().view(np.float32))


@pytest.mark.parametrize("bank", ["a", "b"])
def test_device_bank_reproduces_reference(bank):
    """Trees bit-identical after every append and update; leaves set by update_priorities within 1 ulp of np.power
    (checked before the exact tree comparison); the rest as in tests/test_replay.py."""
    d = rc.load()
    M, C, L, _, _ = rc.config(d, bank)
    be = BankBackend(M, C, L, float(d["discount"]), int(d["n"]), float(d["beta0"]), float(d["omega"]))
    rc.check_bank(d, bank, be, leaf_ulp=1)


def _compare(got, want, where):
    for name in ("tree_idx", "states", "actions", "next_states", "nonterminals", "returns"):
        np.testing.assert_array_equal(got[name], want[name], err_msg="%s %s" % (where, name))
    assert rc.ulp_diff(got["weights"], want["weights"]).max() <= 1, where


def _sync_port(bank, port, C):
    """After an update: leaves within 1 ulp of np.power, the internal nodes their exact float32 sums; the port then
    continues from the device's leaves so that later descents compare exactly."""
    tree = bank.tree.cpu().numpy()
    assert rc.ulp_diff(tree[:, C - 1:], port.tree[:, C - 1:]).max() <= 1
    port.tree[:, C - 1:] = tree[:, C - 1:]
    for i in range(C - 2, -1, -1):
        port.tree[:, i] = port.tree[:, 2 * i + 1] + port.tree[:, 2 * i + 2]
    np.testing.assert_array_equal(tree, port.tree)
    port.max[:] = bank.state.cpu().numpy()[:, 3].copy().view(np.float32)


def test_4096_bins_from_gpu_vec_env_match_port():
    """N = 4096 BlockOut bins, C = 24, obs 3533: ~200 iterations of random valid actions; appends alternate between
    append_from_env and append_batch with a random quarter of the bins marked invalid; every 4th iteration a batch of
    64 (64 distinct memories, one sample each, weights 1) with the bank's own uniforms and one with injected ones,
    then a priority update.  Everything equals the port run on the same data."""
    import torch
    from irbpp_b200 import shapes, learner_glue as glue
    from irbpp_b200.vec_env import GpuVecEnv
    from oracle.replay_port import ReplayPort, replay_uniforms
    dev = _dev()
    N, C, SEL, iters = 4096, 24, 500, 200
    env = GpuVecEnv(shapes.make_blockout_library(32, seed=1), None, num_envs=N, device=dev, item_seed=3)
    L = env.obs_len
    assert L == 3533
    bank = glue.PrioritizedReplayBank(N, C, L, dev, seed=17, max_attempts=4096)
    port = ReplayPort(N, C, L)
    gen = torch.Generator(device=dev); gen.manual_seed(0)
    rng = np.random.default_rng(1)
    state = env.reset()
    n_invalid = n_batches = 0
    for it in range(iters):
        mask = glue.get_mask_from_state(state, SEL)
        q = torch.rand(mask.shape, device=dev, generator=gen)
        q[(1 - mask).bool()] = -float("inf")
        action = q.argmax(1)
        next_state, reward, done, infos = env.step(action.cpu().numpy())
        valid = infos.valid_array().astype(bool)
        s_host, a_host = state.cpu().numpy(), action.cpu().numpy()
        if it % 2 == 0:
            bank.append_from_env(env, state, action, reward_clip=1.0)
        else:
            valid = valid & (rng.random(N) < 0.75)
            bank.append_batch(state, a_host, np.asarray(reward, np.float32).reshape(-1), np.asarray(done).reshape(-1),
                              valid, reward_clip=1.0)
        n_invalid += int((~valid).sum())
        port.append(s_host, a_host, np.asarray(reward, np.float32).reshape(-1), np.asarray(done).reshape(-1), valid, 1.0)
        if it >= 40 and it % 4 == 0:
            bank.anneal_priority_weight(0.01)
            port.priority_weight = bank.priority_weight
            calls = bank.calls
            res = bank.sample(64)
            ids = res[7].cpu().numpy()
            assert len(set(ids.tolist())) == 64
            want = port.sample(ids, 1, replay_uniforms(17, calls, 64, 4096))
            names = ("tree_idx", "states", "actions", "returns", "next_states", "nonterminals", "weights")
            got = {n: res[i].cpu().numpy() if "states" in n else res[i].cpu().numpy().reshape(-1) for i, n in enumerate(names)}
            _compare(got, want, "iteration %d" % it)
            assert (got["weights"] == 1).all()
            loss = torch.rand(64, device=dev, generator=gen) * 2
            bank.update_priorities(res[0], res[7], loss)
            port.update_priorities(ids, got["tree_idx"], loss.cpu().numpy())
            _sync_port(bank, port, C)
            # injected uniforms on memories 0..31, k = 2 (the N <= batch form of the call)
            U = rng.random((64, 64))
            ids2 = torch.arange(32, dtype=torch.int32, device=dev)
            res2 = bank._sample(ids2, 2, torch.from_numpy(U).to(dev))
            want2 = port.sample(np.arange(32), 2, U)
            got2 = {n: res2[i].cpu().numpy() if "states" in n else res2[i].cpu().numpy().reshape(-1) for i, n in enumerate(names)}
            _compare(got2, want2, "iteration %d, injected" % it)
            n_batches += 1
        state = next_state
    torch.cuda.synchronize()
    np.testing.assert_array_equal(bank.tree.cpu().numpy(), port.tree)
    st = bank.state.cpu().numpy()
    np.testing.assert_array_equal(st[:, 0], port.index)
    np.testing.assert_array_equal(st[:, 1], port.full)
    np.testing.assert_array_equal(st[:, 2], port.t)
    np.testing.assert_array_equal(bank.states.cpu().numpy(), port.states)
    np.testing.assert_array_equal(bank.rewards.cpu().numpy(), port.rewards)
    np.testing.assert_array_equal(bank.nonterminals.cpu().numpy(), port.nonterminals)
    assert port.full.all() and n_invalid > 0 and n_batches >= 30
    env.close()


def test_order_level_bank_width():
    """The hierarchical trainer's order-level memory: observation k + 1024 (k = 5), 256 memories, C = 20, with
    terminals, invalid appends, wrap-around and k = 3 strata per memory (N <= batch size)."""
    import torch
    from irbpp_b200.learner_glue import PrioritizedReplayBank
    from oracle.replay_port import ReplayPort, replay_uniforms
    dev = _dev()
    M, C, L = 256, 20, 5 + 1024
    bank, port = PrioritizedReplayBank(M, C, L, dev, seed=3), ReplayPort(M, C, L)
    rng = np.random.default_rng(2)
    for it in range(60):
        obs = rng.random((M, L + 7)).astype(np.float32)
        a, r, d, v = rng.integers(0, 5, M), rng.standard_normal(M).astype(np.float32), rng.random(M) < 0.1, rng.random(M) < 0.9
        bank.append_batch(torch.from_numpy(obs).to(dev)[:, :L], a, r, d, v)       # a strided observation view
        port.append(obs[:, :L], a, r, d, v)
        if it >= 30 and it % 5 == 0:
            calls = bank.calls
            res = bank.sample(3 * M)
            want = port.sample(np.arange(M), 3, replay_uniforms(3, calls, 3 * M, bank.max_attempts))
            names = ("tree_idx", "states", "actions", "returns", "next_states", "nonterminals", "weights")
            got = {n: res[i].cpu().numpy() if "states" in n else res[i].cpu().numpy().reshape(-1) for i, n in enumerate(names)}
            _compare(got, want, "iteration %d" % it)
            np.testing.assert_array_equal(res[7].cpu().numpy(), np.repeat(np.arange(M), 3))
            loss = rng.random(3 * M).astype(np.float32)
            bank.update_priorities(res[0], res[7], torch.from_numpy(loss).to(dev))
            port.update_priorities(np.repeat(np.arange(M), 3), got["tree_idx"], loss)
            _sync_port(bank, port, C)


def test_starved_stratum_raises():
    """C = 16, twelve appends, n = 3, four strata: the reference loops forever; the bank raises naming memory 1."""
    import torch
    from irbpp_b200.learner_glue import PrioritizedReplayBank
    dev = _dev()
    bank = PrioritizedReplayBank(2, 16, 5, dev, multi_step=3, max_attempts=64)
    for k in range(20):
        valid = np.array([True, k < 12])         # memory 1 stops at the probed twelve appends
        bank.append_batch(torch.full((2, 5), float(k), device=dev), [k % 4] * 2, [0.5 * k] * 2, [k % 5 == 4] * 2, valid)
    with pytest.raises(RuntimeError, match=r"memory \[1\]"):
        bank.sample(8)
    for k in range(8):
        bank.append_batch(torch.zeros((2, 5), device=dev), [0, 0], [0.0, 0.0], [False, False])
    bank.sample(8)                               # the error word was cleared; with 20 appends every stratum is served
