"""Batched evaluation over test trajectories: the protocol of the reference's ``tools.test`` (buffer size 1) and
``tools.test_hierachical`` (buffer size k > 1), reference ``tools.py:303-431``, with every trajectory in flight at once.

There one bin plays trajectory 1, 2, ... of ``test_sequence.pt`` (``LoadItemCreator``, ``IRcreator.py:74-101``), one
episode per trajectory.  Here ``num_envs`` bins play them together: bin e plays trajectories ``first + e``,
``first + e + N``, ... (``GpuVecEnv(trajectories=...)``) until none is left, and the per-trajectory results are the
same as the serial loop's."""
import numpy as np

from .vec_env import GpuVecEnv


def evaluate(library, trajectories, policy, num_envs, first=1, count=2000, order_policy=None, **env_kw):
    """Play trajectories ``[first, first + count)`` (``count`` is capped at the trajectories there are) with
    ``num_envs`` bins.

    ``policy(obs) -> actions``: obs is the float32 CUDA tensor ``[N, loc_obs_len]`` of the step (with ``buffer_size``
    k > 1: of ``get_action_candidates``), actions an int64 array or tensor ``[N]`` of candidate rows.  With k > 1,
    ``order_policy(order_obs) -> order actions`` picks the buffered item first (``tools.test_hierachical``).  Actions
    of idle bins are ignored.  ``env_kw`` goes to ``GpuVecEnv`` (``buffer_size``, ``selected_action``, ``device``...).

    Returns a dict: ``trajectory`` (the indices played), per trajectory ``reward_sum``, ``length``, ``ratio``,
    ``counter``, and ``summary``, the figures ``tools.test`` prints: ``avg_reward``, ``avg_length``, ``var_reward``,
    ``var_length``, ``mean_ratio``, ``var_ratio``."""
    k = int(env_kw.get("buffer_size", 1))
    if k > 1 and order_policy is None:
        raise ValueError("buffer_size > 1 needs an order_policy")
    count = max(0, min(int(count), len(trajectories) - int(first)))
    env = GpuVecEnv(library, None, num_envs=num_envs, trajectories=trajectories, first_trajectory=first,
                    num_trajectories=count, **env_kw)
    reward_sum = np.zeros(count, np.float64)
    length = np.zeros(count, np.int64)
    ratio = np.zeros(count, np.float64)
    counter = np.zeros(count, np.int64)
    try:
        obs = env.reset()
        while not env.idle.all():
            playing = env.trajectory.copy()            # step_wait moves finished bins on to their next trajectory
            if k > 1:
                obs = env.get_action_candidates(order_policy(obs), as_tensor=True)
            obs, _, done, infos = env.step(policy(obs))
            if done.any():
                v = infos._views()
                idx = np.nonzero(done)[0]
                t = playing[idx] - first
                reward_sum[t] = v["ep_reward"][idx]   # the episode's rewards summed in float64, as tools.test sums them
                length[t] = v["ep_len"][idx]
                ratio[t] = v["ratio"][idx]
                counter[t] = v["counter"][idx]
    finally:
        env.close()
    summary = {"avg_reward": float(np.mean(reward_sum)), "avg_length": float(np.mean(length)),
               "var_reward": float(np.var(reward_sum)), "var_length": float(np.var(length)),
               "mean_ratio": float(np.mean(ratio)), "var_ratio": float(np.var(ratio))}
    return {"trajectory": np.arange(first, first + count), "reward_sum": reward_sum, "length": length,
            "ratio": ratio, "counter": counter, "summary": summary}
