"""Generate ``item_sources.npz`` from the UNMODIFIED reference item creators.

Run in the build container (needs ``/root/reference`` and torch):

    python tests/golden/make_golden_items.py

It executes reference ``environment/physics0/IRcreator.py`` verbatim (it imports only numpy, copy and torch) and
stores what its classes compute:

* the group tables of ``RandomInstanceCreator`` (``inverseDict``) and ``RandomCateCreator`` (``objCates``) for
  synthetic id -> file dicts: kitchen-style ``category/name_p.obj`` names, and plain names with one- and two-digit
  pose suffixes (``name[0:-6]`` cuts a two-digit suffix one character short, as the reference does);
* the ids every episode draws from ``LoadItemCreator`` over a ``torch.save``-d synthetic trajectory file, for
  buffer sizes 1 and 3, driven as ``binPhy.PackingGame`` drives its creator (``reset()`` + ``preview(k)``, then per
  placement ``update_item_queue(0)`` + ``preview(k)``), across several resets; ``None`` is stored as -1.

The other fixtures of this directory come from ``make_golden.py`` (their provenance is ``PROVENANCE.txt``) and are not
touched here.  ``item_sources.npz`` as committed was written by this script with numpy 2.3.5 and torch 2.11.
"""
import importlib.util
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402


def load_ircreator():
    path = os.path.join(ref_loader.REFERENCE_ROOT, "environment", "physics0", "IRcreator.py")
    spec = importlib.util.spec_from_file_location("irbpp_ref_IRcreator", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def csr(groups):
    off = np.zeros(len(groups) + 1, np.int32)
    off[1:] = np.cumsum([len(g) for g in groups])
    return off, np.array([int(i) for g in groups for i in g], np.int32)


def kitchen_dict(rng):
    names = []
    for cate, base in (("objects", ["bowl", "mug", "can"]), ("concave", ["cup", "pan"]), ("board", ["plank", "tray"])):
        for b in base:
            for p in range(int(rng.integers(1, 4))):
                names.append("%s/%s_%d.obj" % (cate, b, p))
    order = rng.permutation(len(names))
    return {i: names[j] for i, j in enumerate(order)}


def plain_dict(rng):
    names = []
    for s in range(6):
        for p in range(12 if s == 0 else int(rng.integers(1, 6))):    # shape0: pose suffixes up to _11
            names.append("shape%d_%d.obj" % (s, p))
    order = rng.permutation(len(names))
    return {i: names[j] for i, j in enumerate(order)}


def main():
    ir = load_ircreator()
    rng = np.random.default_rng(20261015)
    out = {}
    for tag, d in (("kitchen", kitchen_dict(rng)), ("plain", plain_dict(rng))):
        keys = np.array(list(d.keys()), np.int32)
        out[tag + "_keys"] = keys
        out[tag + "_names"] = np.array(list(d.values()))
        inst = ir.RandomInstanceCreator(keys, d)
        out[tag + "_instance_offsets"], out[tag + "_instance_members"] = csr(list(inst.inverseDict.values()))
        if tag == "kitchen":
            cate = ir.RandomCateCreator(keys, d)
            out[tag + "_category_offsets"], out[tag + "_category_members"] = csr([cate.objCates[c] for c in cate.categories])

    import torch
    trajs = [[int(v) for v in rng.integers(0, 20, size=int(rng.integers(4, 9)))] for _ in range(8)]
    out["traj_offsets"] = np.concatenate([[0], np.cumsum([len(t) for t in trajs])]).astype(np.int64)
    out["traj_items"] = np.array([v for t in trajs for v in t], np.int32)
    placements = [2, 5, 0, 9, 3]                             # per episode; 9 runs past every trajectory's end
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "test_sequence.pt")
        torch.save(trajs, path)
        for k in (1, 3):
            creator = ir.LoadItemCreator(data_name=path)
            traj_index, draws, draw_off = [], [], [0]
            for p in placements:
                creator.reset()
                n0 = len(creator.item_list)
                creator.preview(k)
                seen = list(creator.item_list[n0:])
                for _ in range(p):
                    creator.update_item_queue(0)
                    before = len(creator.item_list)
                    creator.preview(k)
                    seen.extend(creator.item_list[before:])
                traj_index.append(creator.traj_index)
                draws.extend(-1 if v is None else int(v) for v in seen)
                draw_off.append(len(draws))
            out["load_k%d_traj_index" % k] = np.array(traj_index, np.int32)
            out["load_k%d_draws" % k] = np.array(draws, np.int32)
            out["load_k%d_draw_offsets" % k] = np.array(draw_off, np.int64)
    out["load_placements"] = np.array(placements, np.int32)
    np.savez(os.path.join(HERE, "item_sources.npz"), **out)
    print("wrote item_sources.npz")


if __name__ == "__main__":
    main()
