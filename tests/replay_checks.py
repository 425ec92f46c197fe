"""Shared driver of the ``replay.npz`` fixture (``tests/golden/make_golden_replay.py``): replays one bank's recorded
operations through a replay backend and compares every recorded state and output.

A backend has ``append(state, action, reward, done, valid, clip)``, ``sample(mem_ids, k, uniforms, beta) -> dict``,
``update(mem_ids, tree_idxs, loss)`` and ``snapshot() -> (tree, index, full, t, max)``; ``oracle.replay_port`` is one,
the emulated and the real device kernels are the others."""
import numpy as np

from conftest import GOLDEN  # noqa: F401  (tests/ is on sys.path when pytest runs)


def ulp_diff(a, b):
    """Distance in float32 units in the last place (0 for equal values, +0 == -0)."""
    def key(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))


def load():
    import os
    return dict(np.load(os.path.join(GOLDEN, "replay.npz")))


def config(d, p):
    M, C, L, steps, rounds = (int(x) for x in d[p + "_config"])
    return M, C, L, steps, rounds


def check_bank(d, p, backend, leaf_ulp=0, returns_ulp=2, weights_ulp=4):
    """Replays bank ``p``; trees, indices, t, max, tree indices, states, actions and nonterminals must be exact,
    returns within ``returns_ulp`` and weights within ``weights_ulp`` float32 ulp; leaves set by an update within
    ``leaf_ulp`` of numpy's float32 power (the trees are compared exactly as well)."""
    M, C, L, steps, rounds = config(d, p)
    clip = float(d[p + "_clip"])
    r = 0
    for s in range(steps):
        backend.append(d[p + "_app_state"][s], d[p + "_app_action"][s], d[p + "_app_reward"][s],
                       d[p + "_app_done"][s], d[p + "_app_valid"][s], clip)
        tree, index, full, t, mx = backend.snapshot()
        where = "%s step %d" % (p, s)
        np.testing.assert_array_equal(tree, d[p + "_app_tree"][s], err_msg=where)
        np.testing.assert_array_equal(index, d[p + "_app_index"][s], err_msg=where)
        np.testing.assert_array_equal(full, d[p + "_app_full"][s], err_msg=where)
        np.testing.assert_array_equal(t, d[p + "_app_t"][s], err_msg=where)
        np.testing.assert_array_equal(mx, d[p + "_app_max"][s], err_msg=where)
        q = "%sr%d_" % (p, r)
        if r < rounds and int(d[q + "step"]) == s:
            k = int(d[q + "k"])
            out = backend.sample(np.arange(M, dtype=np.int32), k, d[q + "uniforms"], float(d[q + "beta"]))
            where = "%s round %d" % (p, r)
            assert (out["error"] == 0).all(), where
            np.testing.assert_array_equal(out["attempts"], d[q + "attempts"], err_msg=where)
            for name in ("tree_idx", "states", "actions", "next_states", "nonterminals"):
                np.testing.assert_array_equal(out[name], d[q + name], err_msg="%s %s" % (where, name))
            assert ulp_diff(out["returns"], d[q + "returns"]).max() <= returns_ulp, where
            assert ulp_diff(out["weights"], d[q + "weights"]).max() <= weights_ulp, (where, out["weights"], d[q + "weights"])
            backend.update(d[q + "upd_mem"], d[q + "upd_idx"], d[q + "upd_loss"])
            tree, index, full, t, mx = backend.snapshot()
            leaves = d[q + "upd_idx"]
            for m in range(M):
                sel = leaves[d[q + "upd_mem"] == m]
                assert ulp_diff(tree[m, sel], d[q + "after_tree"][m, sel]).max() <= leaf_ulp, where
            np.testing.assert_array_equal(tree, d[q + "after_tree"], err_msg=where)
            np.testing.assert_array_equal(mx, d[q + "after_max"], err_msg=where)
            np.testing.assert_array_equal(index, d[q + "after_index"], err_msg=where)
            r += 1
    assert r == rounds


class PortBackend(object):
    """``oracle.replay_port.ReplayPort`` behind the backend interface."""

    def __init__(self, d, p):
        from oracle.replay_port import ReplayPort
        M, C, L, _, _ = config(d, p)
        self.port = ReplayPort(M, C, L, float(d["discount"]), int(d["n"]), float(d["beta0"]), float(d["omega"]))

    def append(self, state, action, reward, done, valid, clip):
        self.port.append(state, action, reward, done, valid, clip)

    def sample(self, mem_ids, k, uniforms, beta):
        return self.port.sample(mem_ids, k, uniforms, beta)

    def update(self, mem_ids, tree_idxs, loss):
        assert self.port.update_priorities(mem_ids, tree_idxs, loss) == 0

    def snapshot(self):
        return (self.port.tree.copy(),) + self.port.state_block()
