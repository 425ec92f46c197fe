"""Item sources beside sequences and the uniform generator: grouped draws (RandomInstanceCreator /
RandomCateCreator) and trajectory replay (LoadItemCreator), reference ``environment/physics0/IRcreator.py``.

CPU tests: the host helpers against ``golden/item_sources.npz`` (made by ``golden/make_golden_items.py`` from the
unmodified reference classes), and the kernels under the host emulator (``test_kernels_emulated.build_emulated``)
against the Python mirror of the grouped stream and against the oracle, one ``OracleEnv`` per trajectory."""
import ctypes

import numpy as np
import pytest

from conftest import load_golden
from irbpp_b200 import _lib
from test_kernels_emulated import EmuEnv, build_emulated

pytestmark = pytest.mark.timeout(900)

EINVAL, EDEVICE = -1, -4


def _P(a):
    return ctypes.c_void_p(a.ctypes.data)


def _ragged(values, offsets):
    return [list(values[offsets[i]:offsets[i + 1]]) for i in range(len(offsets) - 1)]


# ---- host helpers vs the reference classes ----

@pytest.mark.parametrize("tag", ["kitchen", "plain"])
def test_instance_groups_match_reference(tag):
    from irbpp_b200 import shapes
    d = load_golden("item_sources")
    id2shape = {int(k): str(n) for k, n in zip(d[tag + "_keys"], d[tag + "_names"])}
    off, mem = shapes.group_table(shapes.instance_groups(id2shape))
    assert np.array_equal(off, d[tag + "_instance_offsets"]) and np.array_equal(mem, d[tag + "_instance_members"])


def test_category_groups_match_reference():
    from irbpp_b200 import shapes
    d = load_golden("item_sources")
    id2shape = {int(k): str(n) for k, n in zip(d["kitchen_keys"], d["kitchen_names"])}
    off, mem = shapes.group_table(shapes.category_groups(id2shape))
    assert np.array_equal(off, d["kitchen_category_offsets"]) and np.array_equal(mem, d["kitchen_category_members"])
    with pytest.raises(ValueError):
        shapes.category_groups({k: v for k, v in id2shape.items() if not v.startswith("board/")})


@pytest.mark.parametrize("k", [1, 3])
def test_trajectory_rule_matches_load_item_creator(k):
    """Episode j of a single bin plays trajectory 1 + j from item 0, every draw takes the next item: what
    LoadItemCreator gives under binPhy's reset / preview / update_item_queue protocol, up to its first None."""
    d = load_golden("item_sources")
    trajs = _ragged(d["traj_items"], d["traj_offsets"])
    eps = _ragged(d["load_k%d_draws" % k], d["load_k%d_draw_offsets" % k])
    for j, (t, drawn) in enumerate(zip(d["load_k%d_traj_index" % k], eps)):
        assert t == 1 + j
        n = len(drawn)
        want = (trajs[t] + [-1] * n)[:n]
        assert drawn == want, j


def test_item_group_ids_mirror_is_uniform_per_group():
    from irbpp_b200 import shapes
    groups = [[0], [1, 2, 3], [4, 5]]
    ids = shapes.item_group_ids(7, 64, 400, groups)
    g = np.select([ids == 0, ids <= 3], [0, 1], 2)
    counts = np.bincount(g.reshape(-1), minlength=3) / ids.size
    assert np.all(np.abs(counts - 1 / 3) < 0.01)
    assert np.array_equal(ids[:, :5], shapes.item_group_ids(7, 64, 5, groups))


# ---- kernels under the host emulator ----

@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emulated(str(tmp_path_factory.mktemp("emu_items")))


class ItemEnv(EmuEnv):
    """EmuEnv whose item source is replaced by groups or trajectories; step() also returns Valid."""

    def __init__(self, lib, library, n, groups=None, trajectories=None, first=1, count=None, seed=0, **kw):
        EmuEnv.__init__(self, lib, library, np.zeros((n, 4), np.int32), **kw)
        from irbpp_b200 import shapes
        if groups is not None:
            off, mem = shapes.group_table(groups)
            assert lib.emu_irbpp_set_item_groups(self.h, ctypes.c_uint64(seed), len(groups), _P(off), _P(mem)) == 0
        if trajectories is not None:
            items, off = shapes.trajectory_table(trajectories)
            count = len(trajectories) - first if count is None else count
            assert lib.emu_irbpp_set_trajectories(self.h, _P(items), _P(off), len(trajectories), first, count) == 0

    def step_full(self, actions):
        acts = np.ascontiguousarray(actions, dtype=np.int64)
        obs = np.zeros((self.n, self.obs_len), np.float32)
        assert self.lib.emu_irbpp_step_async(self.h, _P(acts), 0, _P(obs), None) == 0
        res = _lib.IrbppStepResult()
        rc = self.lib.emu_irbpp_step_wait(self.h, ctypes.byref(res))
        view = lambda p, ct, dt: np.frombuffer((ct * self.n).from_address(p), dtype=dt).copy()
        out = {k: view(getattr(res, k), ct, dt) for k, ct, dt in (
            ("reward", ctypes.c_float, np.float32), ("done", ctypes.c_uint8, np.bool_), ("valid", ctypes.c_uint8, np.bool_),
            ("error", ctypes.c_uint8, np.uint8), ("counter", ctypes.c_int32, np.int32), ("ratio", ctypes.c_double, np.float64))}
        return rc, obs, out


def first_valid(obs_row, sel=500):
    v = np.nonzero(np.asarray(obs_row[:sel * 5]).reshape(sel, 5)[:, 4] == 1)[0]
    return int(v[0]) if len(v) else 0


def test_emulated_grouped_stream_matches_mirror(emu):
    """Grouped draws: the episodes equal the oracle fed the mirrored stream (shapes.item_group_ids)."""
    from irbpp_b200 import shapes
    from oracle.oracle_env import OracleConfig, OracleVecEnv
    lib = shapes.make_blockout_library(12, seed=5)
    groups = [[0, 1, 2, 3, 4, 5, 6], [7], [8, 9], [10, 11]]
    n, steps, seed = 5, 8, 99
    env = ItemEnv(emu, lib, n, groups=groups, seed=seed)
    stream = shapes.item_group_ids(seed, n, 4 * steps + 8, groups)
    ora = OracleVecEnv(OracleConfig(ZRotNum=4), lib, stream)
    o = ora.reset()
    assert np.array_equal(env.reset(), o.astype(np.float32))
    for t in range(steps):
        acts = np.array([first_valid(o[i]) for i in range(n)], np.int64)
        o, _, odone, _ = ora.step(acts)
        rc, g, res = env.step_full(acts)
        assert rc == 0 and np.array_equal(g, o.astype(np.float32)), t
        assert np.array_equal(res["done"], odone)
    cursor = np.zeros(n, np.int32)
    assert emu.emu_irbpp_debug_state(env.h, None, None, _P(cursor), None) == 0
    assert np.array_equal(cursor, [e.cursor for e in ora.envs])
    env.close()


def run_trajectories_vs_oracle(make_env, lib, trajs, n, first, count, k, policy, order_policy, heuristics=None):
    """Drive a trajectory-mode env (``make_env()`` -> object with reset / step_full / get_action_candidates) until
    every bin is idle and check every observation and result against one OracleEnv per trajectory.  Returns the
    per-trajectory (reward sum, length, ratio, counter) of the oracle episodes."""
    from oracle.oracle_env import OracleConfig, OracleEnv
    cfg = OracleConfig(ZRotNum=lib.num_rotations, bufferSize=k)
    end = first + count
    env = make_env()
    obs_len = cfg.obs_len
    cur = {}
    per_traj = {}

    def start(e, t):
        if t >= end:
            cur[e] = None
            return np.zeros(obs_len)
        o = OracleEnv(cfg, lib, trajs[t])
        cur[e] = [t, o, 0.0, 0]
        return o.reset()

    want = np.stack([start(e, first + e) for e in range(n)])
    nxt = {e: first + e + n for e in range(n)}
    obs = env.reset()
    assert np.array_equal(obs, want.astype(np.float32))
    steps = 0
    while any(c is not None for c in cur.values()):
        steps += 1
        assert steps < 2000
        if k > 1:
            order = np.array([order_policy(obs[e]) for e in range(n)], np.int64)
            order[[e for e in range(n) if cur[e] is None]] = 99            # ignored by idle bins
            loc = env.get_action_candidates(order)
            for e in range(n):
                w = np.zeros(cfg.loc_obs_len) if cur[e] is None else cur[e][1].get_action_candidates(int(order[e]))
                assert np.array_equal(loc[e], w.astype(np.float32)), (steps, e)
            src = loc
        else:
            src = obs
        acts = np.array([policy(src[e]) for e in range(n)], np.int64)
        acts[[e for e in range(n) if cur[e] is None]] = -5                 # out of range: ignored by idle bins
        rc, obs, res = env.step_full(acts)
        assert rc == 0
        for e in range(n):
            if cur[e] is None:
                assert not res["done"][e] and not res["valid"][e] and res["reward"][e] == 0 and res["error"][e] == 0
                want[e] = 0
                continue
            t, o, rsum, ln = cur[e]
            ob, r, d, info = o.step(int(acts[e]))
            assert res["valid"][e] and np.float32(r) == res["reward"][e] and bool(d) == bool(res["done"][e]), (steps, e)
            cur[e][2] += r
            cur[e][3] += 1
            if d:
                assert res["counter"][e] == info["counter"] and res["ratio"][e] == info["ratio"]
                per_traj[t] = (cur[e][2], cur[e][3], info["ratio"], info["counter"])
                ob = start(e, nxt[e])
                if nxt[e] < end:
                    nxt[e] += n
            want[e] = ob
        assert np.array_equal(obs, want.astype(np.float32)), steps
        if heuristics is not None and k == 1:
            heuristics(env, [cur[e] is None for e in range(n)])
    assert sorted(per_traj) == list(range(first, end))
    return env, per_traj


@pytest.mark.parametrize("k", [1, 5])
def test_emulated_trajectories_match_oracle_until_idle(emu, k):
    """N = 6 bins over a window of 20 trajectories: episode j of bin e plays first + e + 6 j; the run goes on until
    every bin is idle (zero rows, reward 0, done 0, Valid 0, actions ignored, heuristic index -1)."""
    from irbpp_b200 import shapes
    lib = shapes.make_blockout_library(10, seed=8, edge=0.08)
    rng = np.random.default_rng(k)
    trajs = [list(rng.integers(0, lib.num_shapes, size=int(rng.integers(30, 40)))) for _ in range(23)]
    n, first, count = 6, 1, 20

    def check_heuristics(env, idle):
        poses, index = np.zeros((n, 3), np.int32), np.zeros(n, np.int64)
        assert emu.emu_irbpp_heuristic_actions(env.h, 0, 0, _P(poses), _P(index), 0, None) == 0
        assert all(index[e] == -1 for e in range(n) if idle[e])
        assert all(index[e] >= -1 for e in range(n))

    env, per_traj = run_trajectories_vs_oracle(
        lambda: ItemEnv(emu, lib, n, trajectories=trajs, first=first, count=count, buffer_size=k), lib, trajs, n, first,
        count, k, first_valid, lambda row: int(np.argmax(row[:k])), check_heuristics)
    # a reset of idle bins leaves them idle
    obs = env.reset()
    assert not obs.any()
    env.close()


def test_emulated_trajectory_end_is_error_5(emu):
    from irbpp_b200 import shapes
    lib = shapes.make_blockout_library(10, seed=8)
    env = ItemEnv(emu, lib, 3, trajectories=[[1, 2, 3, 4, 5, 6], [1, 2], [3, 4, 5, 6, 7, 8]], first=0)
    obs = env.reset()
    acts = np.array([first_valid(obs[i]) for i in range(3)], np.int64)
    rc, obs, res = env.step_full(acts)            # bin 1 draws its second and last item
    assert rc == 0
    acts = np.array([first_valid(obs[i]) for i in range(3)], np.int64)
    rc, obs, res = env.step_full(acts)
    assert rc == EDEVICE and list(res["error"]) == [0, 5, 0]
    emu.emu_irbpp_last_error.restype = ctypes.c_char_p
    assert b"env 1 reported device error code 5" in emu.emu_irbpp_last_error(env.h)
    env.close()


def test_emulated_bad_tables_are_rejected(emu):
    from irbpp_b200 import shapes
    lib = shapes.make_blockout_library(10, seed=8)
    env = EmuEnv(emu, lib, np.zeros((2, 4), np.int32))
    U = ctypes.c_uint64(1)

    def groups(off, mem):
        off, mem = np.asarray(off, np.int32), np.asarray(mem, np.int32)
        return emu.emu_irbpp_set_item_groups(env.h, U, len(off) - 1, _P(off), _P(mem))

    assert groups([0, 2, 3], [1, 2, 3]) == 0
    assert groups([0, 2, 2, 3], [1, 2, 3]) == EINVAL          # empty group
    assert groups([0, 2, 1], [1, 2, 3]) == EINVAL             # offsets decrease
    assert groups([1, 2, 3], [1, 2, 3]) == EINVAL             # offsets[0] != 0
    assert groups([0, 2, 3], [1, 10, 3]) == EINVAL            # id out of range
    assert groups([0, 2, 3], [1, -1, 3]) == EINVAL

    def trajs(items, off, first, count):
        items, off = np.asarray(items, np.int32), np.asarray(off, np.int64)
        return emu.emu_irbpp_set_trajectories(env.h, _P(items), _P(off), len(off) - 1, first, count)

    assert trajs([1, 2, 3, 4], [0, 2, 4], 0, 2) == 0
    assert trajs([1, 2, 3, 4], [0, 3, 2], 0, 2) == EINVAL     # offsets decrease
    assert trajs([1, 2, 3, 4], [0, 2, 4], 1, 2) == EINVAL     # window outside the pool
    assert trajs([1, 2, 3, 4], [0, 2, 4], -1, 1) == EINVAL
    assert trajs([1, 2, 10, 4], [0, 2, 4], 0, 2) == EINVAL    # id out of range
    assert trajs([1, 2, 3, 4], [0, 0, 4], 0, 2) == EINVAL     # a trajectory of the window with no item for the reset
    assert trajs([1, 2, 3, 4], [0, 0, 4], 1, 1) == 0          # ... outside the window it is never played
    env.close()
