"""The single-environment surface the reference's evaluation loop uses (``tools.test``, reference
``tools.py:303-358``; ``make_eval_env``): ``reset()``, ``step(int)``, ``get_ratio()``, ``get_action_candidates(int)``,
``.packed``, ``.item_creator.traj_index``, ``close()`` -- served by a one-bin ``GpuVecEnv``.

Differences a caller can see, both consequences of DESIGN.md section 1: ``packed`` rows are ``[item id, rotIdx, lx, ly,
z]`` (the pose the placement used; the reference stores PyBullet positions / orientations, and the physics settle is
out of scope), and observations are float32 NumPy rows (the reference returns float64 and ``tools.test`` casts them
to float32 at once, ``tools.py:317``).

The library resets a bin inside the step that ends its episode (the vector-env convention,
``shmem_vec_env.py:140-144``); ``tools.test`` calls ``env.reset()`` itself after ``done``.  So that both draw the same
item stream, the ``reset()`` that follows a finished episode returns the observation the library already produced
instead of resetting (and drawing) a second time."""
import numpy as np

from .vec_env import GpuVecEnv


class _ItemCreatorView(object):
    def __init__(self):
        # LoadItemCreator.traj_index (IRcreator.py:78-92): with trajectories, the one the current episode plays
        # (first_trajectory, first_trajectory + 1, ...); otherwise the number of episodes started so far
        self.traj_index = 0


class SingleGpuEnv(object):
    """``trajectories`` (a list of id lists, ``shapes.load_trajectories``) replays them as ``LoadItemCreator`` does:
    every ``reset()`` moves to the next one, starting at ``first_trajectory`` (1, as ``tools.test`` plays them)."""

    def __init__(self, library, sequence=None, trajectories=None, first_trajectory=1, **kw):
        seqs = None if sequence is None else np.asarray(sequence, dtype=np.int32).reshape(1, -1)
        if trajectories is not None:
            kw.update(trajectories=trajectories, first_trajectory=first_trajectory)
        self._venv = GpuVecEnv(library, seqs, num_envs=1, **kw)
        self._replay = trajectories is not None
        self.library = library
        self.obs_len = self._venv.obs_len
        self.observation_space, self.action_space = self._venv.observation_space, self._venv.action_space
        self.item_creator = _ItemCreatorView()
        self.packed = []
        self._binvol = float(np.prod(np.asarray(self._venv._cfg.bin_dimension[:3], dtype=np.float64)))
        self._pending_reset_obs = None
        self._last = None            # last location observation (candidate rows + next item), host float32

    def reset(self):
        if self._pending_reset_obs is not None:             # the episode ended inside the last step: already reset
            obs, self._pending_reset_obs = self._pending_reset_obs, None
        else:
            obs = self._venv.reset().cpu().numpy()[0]
        self.packed = []
        if self._replay:
            self.item_creator.traj_index = int(self._venv.trajectory[0])
        else:
            self.item_creator.traj_index += 1
        if self._venv.buffer_size == 1:
            self._last = obs
        return obs

    def get_action_candidates(self, orderAction):          # binPhy.py:161-169
        loc = self._venv.get_action_candidates(np.array([int(orderAction)], dtype=np.int64), as_tensor=True).cpu().numpy()[0]
        self._last = loc
        return loc

    def step(self, action):
        a = int(action)
        sel = self._venv.selected_action
        row = self._last[a * 5:a * 5 + 5] if (self._last is not None and 0 <= a < sel) else None
        item = int(self._last[sel * 5]) if self._last is not None else -1
        obs, reward, done, infos = self._venv.step(np.array([a], dtype=np.int64))
        obs = obs.cpu().numpy()[0]
        info = infos[0]
        if done[0]:
            self._final_ratio = info["ratio"]
            self._pending_reset_obs = obs                   # what reset() will hand out
        else:
            if row is not None:
                self.packed.append([item, int(row[0]), int(row[1]), int(row[2]), float(row[3])])
            self._final_ratio = None
            if self._venv.buffer_size == 1:
                self._last = obs
        return obs, float(reward[0, 0]), bool(done[0]), info

    def get_ratio(self):                                    # binPhy.py:149-153
        if getattr(self, "_final_ratio", None) is not None:
            return self._final_ratio                        # the episode that just ended (tools.py:326-327 asks before reset())
        total = 0
        for rec in self.packed:
            total += self.library.volume[rec[0]]
        return total / self._binvol

    def close(self):
        self._venv.close()
