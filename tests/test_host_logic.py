"""Host-side logic of GpuVecEnv that needs no GPU: the single-copy result block, its typed views and
the lazily built info dicts (the reference's per-env dicts: binPhy.py:306-309, monitor.py:58-75)."""

import numpy as np
import pytest

from irbpp_b200 import _lib
from irbpp_b200.vec_env import GpuVecEnv, LazyInfos


def _fake_result(n):
    """A host buffer laid out like the library's pinned result block (include/irbpp.h, irbpp_step_result)."""
    offs, o = {}, 0
    for k, dt in _lib.RESULT_FIELDS:
        offs[k] = o
        o += dt.itemsize * n
    buf = np.zeros(o + 16, np.uint8)
    res = _lib.IrbppStepResult()
    for k in offs:
        setattr(res, k, buf.ctypes.data + offs[k])
    return buf, offs, res


@pytest.mark.parametrize("n", [1, 37, 4096])
def test_result_block_views_and_lazy_infos(n):
    buf, offs, res = _fake_result(n)
    buf[offs["ratio"]:offs["ratio"] + 8 * n].view(np.float64)[:] = np.arange(n) * 0.5
    buf[offs["ep_reward"]:offs["ep_reward"] + 8 * n].view(np.float64)[:] = np.arange(n) * 1.2345678
    buf[offs["reward"]:offs["reward"] + 4 * n].view(np.float32)[:] = np.arange(n)
    buf[offs["counter"]:offs["counter"] + 4 * n].view(np.int32)[:] = np.arange(n) + 100
    buf[offs["ep_len"]:offs["ep_len"] + 4 * n].view(np.int32)[:] = np.arange(n) + 7
    buf[offs["done"]:offs["done"] + n] = np.arange(n) % 2
    buf[offs["valid"]:offs["valid"] + n] = 1
    env = object.__new__(GpuVecEnv)          # no handle: only the pure-host helpers are exercised
    env.num_envs = n
    src, got_offs = env._result_block(res)
    assert got_offs == offs and src.ctypes.data == buf.ctypes.data
    assert env._result_block(res)[0] is src                       # built once per block
    block = src.copy()
    done = block[offs["done"]:offs["done"] + n].view(np.bool_)
    infos = LazyInfos(n, block, offs, done, 1.5)
    borrowed = LazyInfos(n, src, offs, done.copy(), 1.5, borrowed=True)   # as step_wait builds it: a view of the pinned block ...
    borrowed.detach()                                                     # ... copied before the library reuses the block
    buf[:] = 0                                                    # the step's copy is private
    assert borrowed[n - 1] == infos[n - 1] and borrowed.finished()[1].tolist() == infos.finished()[1].tolist()
    assert len(infos) == n
    assert infos[0] == {"Valid": True}
    if n > 1:
        i = n - 1 if (n - 1) % 2 else n - 2
        assert infos[i] == {"Valid": True, "counter": 100 + i, "ratio": 0.5 * i,
                            "episode": {"r": round(1.2345678 * i, 6), "l": 7 + i, "t": 1.5}}
        assert infos[-1] == infos[n - 1]
        assert [d["Valid"] for d in infos[0:2]] == [True, True]
    with pytest.raises(IndexError):
        infos[n]
    # batched views (learner glue, SURVEY.md 8(f)2): the same numbers without building dicts
    idx, ep_r, ratio, counter, valid = infos.finished()
    assert np.array_equal(idx, np.nonzero(done)[0]) and infos.valid_array().all() and len(infos.valid_array()) == n
    for k, i in enumerate(idx[:4]):
        d = infos[int(i)]
        assert d["episode"]["r"] == ep_r[k] and d["ratio"] == ratio[k] and d["counter"] == counter[k] and valid[k]


def test_learner_glue_host_pieces():
    from irbpp_b200 import learner_glue as glue
    obs = np.arange(3 * 3533, dtype=np.float32).reshape(3, 3533)
    m = glue.get_mask_from_state(obs, 500)
    assert m.shape == (3, 500) and m[2, 7] == obs[2, 7 * 5 + 4]          # tools.py:298-299
    assert glue.segment_size(64, 4) == (4, 16)                           # agent.py:69 when it works
    assert glue.segment_size(64, 4096) == (64, 1)                        # ... and when int(64 / 4096) == 0


class _Ev(object):
    """Stand-in for a CUDA event at a fixed position on the device time line (ms)."""

    def __init__(self, t):
        self.t = t

    def elapsed_time(self, other):
        return other.t - self.t


def test_bench_gather_accounting():
    """bench.py's split of one rollout gather into hidden / beside-flush / tail and the charge derived from it."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    origin = _Ev(0.0)
    # 10 steps of 0.10 ms with 0.05 ms flush gaps; the first three are slowed to 0.12 by the gather [0, 0.45]
    steps, t = [], 0.0
    for i in range(10):
        d = 0.12 if i < 3 else 0.10
        steps.append((_Ev(t), _Ev(t + d)))
        t += d + 0.05
    g, hidden, tail, flush, exposed = bench.gather_account(origin, (_Ev(0.0), _Ev(0.45)), steps, [])
    assert abs(g - 0.45) < 1e-12 and abs(hidden - 0.35) < 1e-9 and tail == 0.0 and abs(flush - 0.10) < 1e-9
    assert abs(exposed - (0.10 / 0.10) * 0.02) < 1e-9           # one further step, 0.02 ms slower
    # a gather that outlasts the rollout: the tail is charged in full
    end = steps[-1][1].t
    g, hidden, tail, flush, exposed = bench.gather_account(origin, (_Ev(end - 0.05), _Ev(end + 0.30)), steps, [])
    assert abs(tail - 0.30) < 1e-9 and abs(hidden - 0.05) < 1e-9 and abs(flush) < 1e-9 and exposed >= 0.30
    # the agent stand-in hides gather time like a step does
    g, hidden, tail, flush, exposed = bench.gather_account(origin, (_Ev(0.12), _Ev(0.17)), steps, [(_Ev(0.12), _Ev(0.17))])
    assert abs(hidden - 0.05) < 1e-9 and abs(exposed) < 1e-9
