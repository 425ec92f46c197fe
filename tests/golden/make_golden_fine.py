"""Generate the 32 x 32 action-grid fixtures (``fine_*.npz``) from the UNMODIFIED reference.

Run in the build container (needs ``/root/reference`` and cv2):

    python tests/golden/make_golden_fine.py

The reference's README trains the Cube dataset with resolutionA = resolutionH = 0.01, i.e. ``stepSize`` 1 and a
32 x 32 action grid.  As ``make_golden.py`` does for the 16 x 16 grid, this script executes reference
``environment/physics0/space.py`` (``Space.get_possible_position``, ``space.py:98-129``; ``Space.get_heuristic_action``,
``space.py:162-227``) and ``environment/physics0/cvTools.py`` (``getConvexHullActions``, ``cvTools.py:61-103``)
verbatim via ``oracle/ref_loader.py``, with ``Space`` constructed at resolutionAct 0.01, and stores their outputs:

* ``fine_scan_cube.npz``, ``fine_scan_irregular.npz``: get_possible_position on random heightmaps;
* ``fine_hulls.npz``: getConvexHullActions on random 32 x 32 maps, including all-masked maps (``None``);
* ``fine_episode_cube.npz`` (Cube boxes, R = 2), ``fine_episode_blockout.npz`` (BlockOut shapes, R = 4,
  selectedAction 40: the truncation of binPhy.py:209-212 fires), ``fine_episode_buffered.npz`` (k = 5);
* ``fine_heuristic.npz``: get_heuristic_action, four methods x four directions, along an episode stepped with them.

Episodes drive the verbatim functions through the restated ``binPhy`` glue of ``oracle/oracle_env.py``
(``RefGeometry`` backend) -- the glue cannot run verbatim (gym / pybullet).  The 16 x 16 fixtures are not touched.
The GPU box has no reference tree; tests there read only the ``.npz`` files written here.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (lib_arrays, random_heightmap, gen_episode of the 16 x 16 fixtures)
from irbpp_b200 import shapes  # noqa: E402
from oracle import ref_loader  # noqa: E402
from oracle.oracle_env import HEURISTICS, OracleConfig, OracleVecEnv, RefGeometry  # noqa: E402

RES_A = 0.01
A = 32


def fine_config(**kw):
    return OracleConfig(resolutionAct=RES_A, **kw)


def gen_scan_cases(space_mod, lib, R, seed):
    cfg = fine_config(ZRotNum=R)
    rng = np.random.default_rng(seed)
    sp = space_mod.Space(cfg.bin_dimension, cfg.resolutionAct, cfg.resolutionH, False, R, lib.shot_info(), [100, 100, 100])
    hms, ids, pz, pv, mk = [], [], [], [], []
    for case in range(16):
        hm = make_golden.random_heightmap(rng, case % 4)
        item = int(rng.integers(0, lib.num_shapes))
        sp.heightmapC = hm
        meshes = [ref_loader.MeshStandIn(lib.extents[item, r]) for r in range(R)]
        mask = sp.get_possible_position(item, meshes, 500)
        hms.append(hm.copy()); ids.append(item)
        pz.append(sp.posZmap.copy()); pv.append(sp.posZValid.copy()); mk.append(mask.copy())
    d = make_golden.lib_arrays(lib)
    d.update(R=np.array(R), heightmaps=np.array(hms), item_ids=np.array(ids), posZmap=np.array(pz),
             posZValid=np.array(pv), naiveMask=np.array(mk))
    return d


def gen_hull_cases(cv_mod):
    """Random [32, 32] posZValid / mask maps -> rows [rot, row, col, H, V] of the verbatim getConvexHullActions (counts 0:
    it returned None)."""
    rng = np.random.default_rng(17)
    posz, masks, rows, counts = [], [], [], []
    for case in range(48):
        kind = case % 4
        if kind == 0:    # blocky levels
            lv = np.zeros((A, A))
            for _ in range(int(rng.integers(1, 14))):
                x0, y0 = rng.integers(0, A - 1, size=2); w, h = rng.integers(1, 17, size=2)
                lv[x0:x0 + w, y0:y0 + h] = rng.integers(0, 8)
            pz = lv * 0.04
        elif kind == 1:  # noisy multiples of 0.01 (floor-divide hazards)
            pz = rng.integers(0, 31, size=(A, A)) * 0.01
        elif kind == 2:  # arbitrary floats incl. negatives
            pz = rng.uniform(-0.05, 0.3, size=(A, A))
        else:            # few levels, big regions with holes: long borders
            pz = (rng.random((A, A)) < 0.35) * 0.05 + (rng.random((A, A)) < 0.2) * 0.02
        mask = (rng.random((A, A)) > (0.1 if case % 8 < 6 else 0.6)).astype(np.float64)
        if case % 12 == 11:
            mask[:] = 0  # no candidate at all: None
        pv = np.where(mask == 1, pz, 1e3)
        res = cv_mod.getConvexHullActions(pv[None], mask[None], 0.01)
        posz.append(pv); masks.append(mask)
        if res is None:
            counts.append(0)
        else:
            counts.append(len(res)); rows.append(res)
    return dict(posZValid=np.array(posz), mask=np.array(masks), counts=np.array(counts),
                rows=np.concatenate(rows, axis=0))


def gen_episode(tag, lib, R, n_envs, n_steps, seed, **kw):
    """make_golden.gen_episode with the configurations at resolutionAct 0.01 (it builds its OracleConfig by name)."""
    make_golden.OracleConfig = fine_config
    try:
        return make_golden.gen_episode(tag, lib, R, n_envs, n_steps, seed, **kw)
    finally:
        make_golden.OracleConfig = OracleConfig


def gen_heuristic_episode(lib, R, n_envs, n_steps, seed):
    """As make_golden.gen_heuristic_episode, poses flattened on the 32 x 32 grid."""
    cfg = fine_config(ZRotNum=R)
    seqs = shapes.make_sequences(n_envs, 48, lib.num_shapes, seed=seed)
    vec = OracleVecEnv(cfg, lib, seqs, lambda c, l: RefGeometry(c, l))
    obs_log = [vec.reset().copy()]
    pose_log, index_log, act_log, rew_log, done_log = [], [], [], [], []
    for t in range(n_steps):
        poses = np.zeros((4, 4, n_envs, 3), np.int32)
        index = np.zeros((4, 4, n_envs), np.int64)
        for mi, m in enumerate(HEURISTICS):
            for d in range(4):
                poses[mi, d], index[mi, d] = vec.heuristic_actions(m, d)
        pose_log.append(poses); index_log.append(index)
        p = poses[t % 4, (t // 4) % 4]
        acts = (p[:, 0].astype(np.int64) * A + p[:, 1]) * A + p[:, 2]
        obs, rew, done, _ = vec.step(acts, poses=True)
        act_log.append(acts); obs_log.append(obs.copy()); rew_log.append(rew); done_log.append(done)
    d = make_golden.lib_arrays(lib)
    d.update(R=np.array(R), sequences=seqs, poses=np.array(pose_log), index=np.array(index_log),
             actions=np.array(act_log), obs=np.array(obs_log).astype(np.float32),
             reward=np.array(rew_log), done=np.array(done_log))
    print("heuristic dones", int(np.sum(done_log)), "not-a-candidate", int((d["index"] < 0).sum()))
    return d


def main():
    assert ref_loader.reference_available(), "needs /root/reference"
    _, space_mod, cv_mod = ref_loader.load_reference()
    out = {
        "fine_scan_cube": gen_scan_cases(space_mod, shapes.make_cube_library(seed=13, num_shapes=12, resolutionAct=RES_A), 2, 31),
        "fine_scan_irregular": gen_scan_cases(space_mod, shapes.make_irregular_library(12, seed=12, num_rotations=2,
                                                                                        resolutionAct=RES_A), 2, 32),
        "fine_hulls": gen_hull_cases(cv_mod),
        "fine_episode_cube": gen_episode("fine-cube", shapes.make_cube_library(seed=3, num_shapes=24, resolutionAct=RES_A),
                                         2, 3, 36, 41),
        "fine_episode_blockout": gen_episode("fine-blockout", shapes.make_blockout_library(16, seed=1, resolutionAct=RES_A),
                                             4, 3, 24, 42, selectedAction=40),
        "fine_episode_buffered": gen_episode("fine-buffered", shapes.make_cube_library(seed=5, num_shapes=24, resolutionAct=RES_A),
                                             2, 2, 16, 43, bufferSize=5),
        "fine_heuristic": gen_heuristic_episode(shapes.make_irregular_library(8, seed=7, num_rotations=2, resolutionAct=RES_A),
                                                2, 2, 10, 44),
    }
    for k, d in out.items():
        np.savez_compressed(os.path.join(HERE, k + ".npz"), **d)
    import cv2
    with open(os.path.join(HERE, "PROVENANCE_FINE.txt"), "w") as f:
        f.write("fine_*.npz generated by tests/golden/make_golden_fine.py from the unmodified reference at %s "
                "(resolutionA = resolutionH = 0.01)\n" % ref_loader.REFERENCE_ROOT)
        f.write("numpy %s, cv2 %s\n" % (np.__version__, cv2.__version__))


if __name__ == "__main__":
    main()
