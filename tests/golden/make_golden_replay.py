"""Generate ``replay.npz`` from the UNMODIFIED reference replay memory.

Run in the build container (needs the reference tree and torch):

    python tests/golden/make_golden_replay.py

It executes reference ``memory.py`` verbatim (it imports only numpy and torch) and drives ``ReplayMemory`` objects
as ``trainer.py`` and ``Agent.learn`` do: per step every memory whose transition is valid appends
``(state, action, reward, done)`` after the reward clamp (``trainer.py:181-186``); every few steps each memory is
sampled with ``sample(k)`` (``agent.py:69-75``), β is annealed (``trainer.py:197``) and priorities are written back
with ``update_priorities`` (``agent.py:123-124``), here with a duplicated tree index and zero losses mixed in.

``np.random.uniform`` is replaced while the reference runs by a function that draws ``U = np.random.random_sample()``
itself and returns ``low + (high - low) * U`` (what ``RandomState.uniform`` computes); before that, the script asserts
that the two return bit-identical values from the same ``RandomState``.  Every ``U`` is recorded, per stratum, so
that the device bank and ``oracle/replay_port.py`` can replay the same draws.

Recorded per bank (prefix ``a_`` / ``b_``): the inputs of every append step, the trees and state blocks after it;
per sample round the k, β, uniforms (padded with 0.5), attempt counts and all seven outputs; the update rows and the
trees / state blocks after them.

Not run here: the reference loops forever on C = 16, twelve appends, n = 3, ``sample(4)`` (stratum 3 covers only
leaves 9-11, which all lie within n of the write index); ``tests/test_replay.py`` checks that the bounded device
version reports that case instead.  ``replay.npz`` as committed was written by this script with numpy 2.3.5 and
torch 2.11.
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402

BANKS = {   # prefix: (M, C, obs_len, steps, reward_clip, k per round, seed)
    "a": (3, 24, 5, 70, 1.0, (4, 1, 4, 4, 1, 4, 4, 1, 4, 4), 11),
    "b": (2, 37, 4, 90, 0.0, (1, 4, 4, 1, 4, 4, 1, 4, 4, 1, 4), 12),
}
N_STEP, DISCOUNT, BETA0, OMEGA, BETA_STEP = 3, 0.99, 0.4, 0.5, 0.07
MAX_ATTEMPTS = 10000


def load_memory():
    path = os.path.join(ref_loader.REFERENCE_ROOT, "memory.py")
    spec = importlib.util.spec_from_file_location("irbpp_ref_memory", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def check_uniform_wrapper(torch):
    a, b = np.random.RandomState(3), np.random.RandomState(3)
    for i in range(2000):
        lo = torch.tensor(np.float32(np.random.RandomState(i).rand() * 10), dtype=torch.float32)
        hi = lo * 2 + 1
        want = a.uniform(lo, hi)
        got = float(lo) + (float(hi) - float(lo)) * b.random_sample()
        assert type(want) is float and np.float64(want).tobytes() == np.float64(got).tobytes(), (i, want, got)


def run_bank(mem_mod, torch, prefix, M, C, L, steps, clip, ks, seed):
    args = types.SimpleNamespace(distributed=False, device=torch.device("cpu"), discount=DISCOUNT, multi_step=N_STEP,
                                 priority_weight=BETA0, priority_exponent=OMEGA)
    mems = [mem_mod.ReplayMemory(args, C, L) for _ in range(M)]
    rng = np.random.default_rng(seed)
    np.random.seed(seed)
    out = {}
    app = {k: [] for k in ("state", "action", "reward", "done", "valid", "tree", "index", "full", "t", "max")}

    def snapshot(d):
        d["tree"].append(np.stack([m.transitions.sum_tree.numpy().copy() for m in mems]))
        d["index"].append(np.array([m.transitions.index.value for m in mems], np.int32))
        d["full"].append(np.array([int(bool(m.transitions.full.value)) for m in mems], np.int32))
        d["t"].append(np.array([m.t for m in mems], np.int32))
        d["max"].append(np.array([float(m.transitions.max) for m in mems], np.float32))

    log = []
    real_uniform = np.random.uniform

    def uniform(low, high):
        u = np.random.random_sample()
        log[-1].append(u)
        if len(log[-1]) > MAX_ATTEMPTS:
            raise RuntimeError("a stratum is starved: choose another configuration")
        return float(low) + (float(high) - float(low)) * u

    rounds, beta = 0, BETA0
    for s in range(steps):
        state = rng.standard_normal((M, L)).astype(np.float32)
        action = rng.integers(0, 500, M)
        reward = (rng.standard_normal(M) * 1.5).astype(np.float32)
        done = rng.random(M) < 0.12
        valid = rng.random(M) < 0.85
        rew_t = torch.from_numpy(reward.copy())
        if clip > 0:
            c = torch.full((M,), clip)
            rew_t = torch.maximum(torch.minimum(rew_t, c), -c)              # trainer.py:181-182
        st_t, act_t = torch.from_numpy(state.copy()), torch.from_numpy(action.copy())
        for i in range(M):
            if valid[i]:
                mems[i].append(st_t[i], act_t[i], rew_t[i], bool(done[i]))   # trainer.py:184-186
        for k_, v in (("state", state), ("action", action), ("reward", reward), ("done", done), ("valid", valid)):
            app[k_].append(v)
        snapshot(app)
        if s >= 25 and s % 4 == 0 and rounds < len(ks):
            k = ks[rounds]
            p = "%sr%d_" % (prefix, rounds)
            beta = min(beta + BETA_STEP, 1.0)                                # trainer.py:197
            samples, unis = [], []
            np.random.uniform = uniform
            try:
                for m in mems:
                    m.priority_weight = beta
                    orig = m._get_sample_from_segment

                    def seg(segment, i, orig=orig):
                        log.append([])
                        return orig(segment, i)
                    m._get_sample_from_segment = seg
                    samples.append(m.sample(k))
                    del m._get_sample_from_segment
                    unis.extend(log[-k:])
            finally:
                np.random.uniform = real_uniform
            A = max(len(u) for u in unis)
            U = np.full((M * k, A), 0.5)
            for r, u in enumerate(unis):
                U[r, :len(u)] = u
            out[p + "k"] = np.int32(k)
            out[p + "step"] = np.int32(s)
            out[p + "beta"] = np.float64(beta)
            out[p + "uniforms"] = U
            out[p + "attempts"] = np.array([len(u) for u in unis], np.int32)
            out[p + "tree_idx"] = np.array([i for smp in samples for i in smp[0]], np.int64)
            for j, name in ((1, "states"), (2, "actions"), (3, "returns"), (4, "next_states"), (5, "nonterminals"),
                            (6, "weights")):
                out[p + name] = torch.cat([smp[j] for smp in samples]).numpy()
            # write-back rows: memory i's k losses (agent.py:123-124); zeros mixed in, and memory 0 gets its first
            # index again with another loss at the end of its rows (the later value must win)
            um, ui, ul = [], [], []
            for i, smp in enumerate(samples):
                loss = (rng.random(k) * 3 + 0.3).astype(np.float32)
                loss[rng.random(k) < 0.15] = 0.0
                idxs = list(smp[0])
                if i == 0:
                    idxs.append(idxs[0])
                    loss = np.append(loss, np.float32(rng.random() * 2 + 0.5))
                mems[i].update_priorities(idxs, torch.from_numpy(loss))
                um += [i] * len(idxs); ui += idxs; ul += list(loss)
            out[p + "upd_mem"] = np.array(um, np.int32)
            out[p + "upd_idx"] = np.array(ui, np.int64)
            out[p + "upd_loss"] = np.array(ul, np.float32)
            upd = {k_: [] for k_ in ("tree", "index", "full", "t", "max")}
            snapshot(upd)
            for k_, v in upd.items():
                out[p + "after_" + k_] = v[0]
            rounds += 1
    assert rounds == len(ks), (prefix, rounds)
    for k_, v in app.items():
        out["%s_app_%s" % (prefix, k_)] = np.stack(v)
    out[prefix + "_config"] = np.array([M, C, L, steps, rounds], np.int32)
    out[prefix + "_clip"] = np.float64(clip)
    return out


def main():
    import torch
    torch.set_num_threads(1)
    check_uniform_wrapper(torch)
    mem_mod = load_memory()
    out = dict(n=np.int32(N_STEP), discount=np.float64(DISCOUNT), omega=np.float64(OMEGA), beta0=np.float64(BETA0))
    for prefix, cfg in BANKS.items():
        out.update(run_bank(mem_mod, torch, prefix, *cfg))
    path = os.path.join(HERE, "replay.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
