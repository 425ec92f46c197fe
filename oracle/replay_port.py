"""NumPy restatement of the reference's prioritized n-step replay (``memory.py:15-208``) for M memories at once.

It keeps the reference's float32 arithmetic step by step, so that the device bank (``csrc/irbpp_replay.cuh``) can be
compared with it at any N without the reference tree.  Two things differ from ``memory.py`` on purpose:

* the uniforms of the stratified draws are INJECTED (``uniforms[row, attempt]``, the ``U`` of
  ``np.random.uniform(lo, hi) = lo + (hi - lo) * U``), and a stratum gives up after ``uniforms.shape[1]`` attempts
  with error code 1 where ``_get_sample_from_segment`` (``:163-170``) would loop forever;
* importance weights use ``float32(float64(x) ** float64(float32(-beta)))``, which is what the device computes;
  torch's float32 ``pow`` (``:201``) can differ from it in the last bits, and the tests state that tolerance.

Actions are stored as int64 (the reference stores them as float32 and returns ``.to(int64)``, exact below 2^24).
"""
import numpy as np

F32 = np.float32
ERR_STARVED, ERR_MEMORY, ERR_INDEX = 1, 2, 3


def _mix(z):
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def replay_uniforms(seed, call, rows, attempts):
    """``rp_uniform`` of ``csrc/irbpp_replay.cuh``: the [rows, attempts] float64 uniforms the device draws when no
    uniforms are supplied (splitmix64 of (seed, call, row, attempt), 53 bits)."""
    gold = np.uint64(0x9E3779B97F4A7C15)
    with np.errstate(over="ignore"):
        z0 = _mix(np.array([seed], np.uint64) + gold * np.array([call + 1], np.uint64))
        r = np.arange(rows, dtype=np.uint64)[:, None]
        a = np.arange(attempts, dtype=np.uint64)[None, :]
        z = _mix(z0 + gold * ((r << np.uint64(16)) + a + np.uint64(1)))
    return (z >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


class ReplayPort(object):
    """M ``ReplayMemory(args, capacity, obs_len)`` objects (``memory.py:95-107``) as memory-major arrays."""

    def __init__(self, num_memories, capacity, obs_len, discount=0.99, multi_step=3, priority_weight=0.4,
                 priority_exponent=0.5):
        M, C, L = int(num_memories), int(capacity), int(obs_len)
        self.M, self.C, self.L, self.n = M, C, L, int(multi_step)
        self.priority_weight, self.priority_exponent = priority_weight, priority_exponent
        self.tree = np.zeros((M, 2 * C - 1), F32)                      # SegmentTree.sum_tree (:29)
        self.states = np.zeros((M, C, L), F32)
        self.timesteps = np.zeros((M, C), np.int32)
        self.actions = np.zeros((M, C), np.int64)
        self.rewards = np.zeros((M, C), F32)
        self.nonterminals = np.zeros((M, C), np.uint8)
        self.index = np.zeros(M, np.int32)
        self.full = np.zeros(M, np.int32)
        self.t = np.zeros(M, np.int32)
        self.max = np.ones(M, F32)                                       # :27
        self.scale = np.array([discount ** i for i in range(self.n)], F32)   # :107

    def state_block(self):
        return self.index.copy(), self.full.copy(), self.t.copy(), self.max.copy()

    def _update(self, m, node, value):
        """SegmentTree.update (:53-56): set the leaf, recompute its ancestors as left + right (:45-50)."""
        tree = self.tree[m]
        tree[node] = value
        i = node
        while i > 0:
            p = (i - 1) // 2
            tree[p] = tree[2 * p + 1] + tree[2 * p + 2]
            i = p
        if self.max[m] > value:                                          # Python max(value, self.max)
            return
        self.max[m] = value

    def append(self, state, action, reward, done, valid=None, reward_clip=0.0):
        """ReplayMemory.append (:110-113, SegmentTree.append :58-69) for every memory with ``valid`` set
        (trainer.py:184-186), after the optional reward clamp of trainer.py:181-182."""
        C = self.C
        for m in range(self.M):
            if valid is not None and not valid[m]:
                continue
            idx = int(self.index[m])
            r = F32(reward[m])
            if reward_clip > 0:
                r = max(min(r, F32(reward_clip)), F32(-reward_clip))
            self.timesteps[m, idx] = self.t[m]
            self.states[m, idx] = state[m]
            self.actions[m, idx] = action[m]
            self.rewards[m, idx] = r
            self.nonterminals[m, idx] = 0 if done[m] else 1
            self._update(m, idx + C - 1, self.max[m])
            self.index[m] = (idx + 1) % C
            self.full[m] = int(bool(self.full[m]) or self.index[m] == 0)
            self.t[m] = 0 if done[m] else self.t[m] + 1

    def _descend(self, m, v):
        """SegmentTree._retrieve (:72-79): compares and subtracts in float32."""
        tree, x, size = self.tree[m], 0, 2 * self.C - 1
        while 2 * x + 1 < size:
            left = tree[2 * x + 1]
            if v <= left:
                x = 2 * x + 1
            else:
                v = F32(v - left)
                x = 2 * x + 2
        return x

    def sample(self, mem_ids, k, uniforms, priority_weight=None):
        """ReplayMemory.sample(k) (:191-203) of every memory in ``mem_ids``; row g * k + i is stratum i of memory
        mem_ids[g].  ``uniforms`` float64 [len(mem_ids) * k, A].  Returns a dict of the device outputs."""
        beta = self.priority_weight if priority_weight is None else priority_weight
        C, L, n = self.C, self.L, self.n
        uniforms = np.asarray(uniforms, np.float64)
        B, A = len(mem_ids) * k, uniforms.shape[1]
        out = dict(tree_idx=np.full(B, -1, np.int64), states=np.zeros((B, L), F32), actions=np.zeros(B, np.int64),
                   returns=np.zeros(B, F32), next_states=np.zeros((B, L), F32), nonterminals=np.zeros(B, F32),
                   weights=np.zeros(B, F32), attempts=np.zeros(B, np.int32), error=np.zeros(B, np.int32))
        neg_beta = float(F32(-beta))
        for g, m in enumerate(mem_ids):
            rows = range(g * k, (g + 1) * k)
            if not 0 <= m < self.M:
                out["error"][list(rows)] = ERR_MEMORY
                continue
            tree, index = self.tree[m], int(self.index[m])
            total = tree[0]
            seg = F32(total / F32(k))                                    # :193
            cap = F32(C if self.full[m] else index)                      # :200
            for i, b in enumerate(rows):
                lo, hi = float(F32(F32(i) * seg)), float(F32(F32(i + 1) * seg))
                node = -1
                for a in range(A):                                       # :165-170, bounded
                    out["attempts"][b] = a + 1
                    x = self._descend(m, F32(lo + (hi - lo) * uniforms[b, a]))
                    idx = x - (C - 1)
                    if (index - idx) % C > n and (idx - index) % C >= 1 and tree[x] != 0:
                        node = x
                        break
                if node < 0:
                    out["error"][b] = ERR_STARVED
                    continue
                idx = node - (C - 1)
                # :115-130: entries idx + t, t = 0..n; after the first fetched terminal, blank transitions
                R, nt, fetch = F32(0), F32(0), True
                for t in range(n + 1):
                    slot = (idx + t) % C
                    rw, nt = F32(0), F32(0)
                    if fetch:
                        rw, nt = self.rewards[m, slot], F32(self.nonterminals[m, slot])
                        if t == n:
                            out["next_states"][b] = self.states[m, slot]
                    if t < n:
                        R = F32(R + F32(rw * self.scale[t]))              # :181-182, summed in order
                    fetch = nt != 0
                out["tree_idx"][b] = node
                out["states"][b] = self.states[m, idx]
                out["actions"][b] = self.actions[m, idx]
                out["returns"][b] = R
                out["nonterminals"][b] = nt
                p = F32(cap * F32(tree[node] / total))                   # :199-201
                out["weights"][b] = F32(float(p) ** neg_beta)
            ok = [b for b in rows if out["error"][b] == 0]
            if ok:
                out["weights"][ok] = out["weights"][ok] / out["weights"][ok].max()   # :202
        return out

    def update_priorities(self, mem_ids, tree_idxs, loss):
        """Agent.learn's write-back (agent.py:123-124) as rows (memory, tree index, loss) in batch order:
        ``np.power(loss, priority_exponent)`` in float32 (:207), then one SegmentTree.update per row (:208)."""
        pri = np.power(np.asarray(loss, F32), self.priority_exponent)
        bad = False
        for m, node, v in zip(mem_ids, tree_idxs, pri):
            if not (0 <= m < self.M and self.C - 1 <= node < 2 * self.C - 1):
                bad = True
                continue
            self._update(int(m), int(node), F32(v))
        return ERR_INDEX if bad else 0
