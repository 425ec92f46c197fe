"""Shape tables: the input format of the packing hot path.

The reference never touches meshes inside ``step``: it consumes per
(shape id, rotation) tables ``(heightMapT, heightMapB, maskT, maskB)`` that
``tools.shotInfoPre`` (reference ``tools.py:248-279``) caches from
``tools.shot_item`` (``tools.py:98-135``), plus ``mesh.extents``
(``space.py:104``) and ``infoDict[id][0]['volume']`` (``binPhy.py:149-156``).
This module holds that format (``ShapeLibrary``) and synthetic generators for
it, because the reference's datasets are a Google-Drive download that is not
available offline (SURVEY.md section 8d):

* ``make_blockout_library``  - voxel polycubes, R = 4 (rot90 about z)
* ``make_cube_library``      - boxes, R = 2
* ``make_irregular_library`` - non-flat bottoms, holes, extents that are not
  multiples of the heightmap resolution, R = 8 (or any R)

Tables are sampled with the ``shot_item`` rule: pixel (i, j) is the ray through
``(i*resH + 0.001, j*resH + 0.001)`` (``tools.py:81-96``); a miss gives height 0
and mask 0.  Window sizes come from the reference formula
``ceil(round(extent, 6) / res)`` (``space.py:104-106``) evaluated in float64 on
the host -- never recomputed in integers (``0.28/0.01 -> 29``).
"""
from dataclasses import dataclass, field
from typing import List, Tuple

import numpy as np

RAY_SHIFT = 0.001  # tools.py:81 (shift = 0.001 passed at space.py:28)


def window_dims(extents, resolutionH, resolutionAct):
    """(w, h, wA, hA) exactly as reference space.py:104-106."""
    boundingSize = np.round(np.asarray(extents, dtype=np.float64), decimals=6)
    w, h = np.ceil(boundingSize[0:2] / resolutionH).astype(np.int32)
    wA, hA = np.ceil(boundingSize[0:2] / resolutionAct).astype(np.int32)
    return int(w), int(h), int(wA), int(hA)


@dataclass
class ShapeLibrary:
    """All shape tables of one dataset.

    ``tables[s][r] = (T, B, mT, mB)`` float64 arrays of shape ``[w, h]`` (the
    reference's ``shotInfo[s][r]``), ``extents[s, r]`` the raw ``mesh.extents``
    of that rotation, ``volume[s]`` the mesh volume.
    """
    resolutionH: float
    resolutionAct: float
    extents: np.ndarray                 # [S, R, 3] float64
    volume: np.ndarray                  # [S] float64
    tables: List[List[Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]]]
    name: str = "synthetic"
    dims: np.ndarray = field(default=None)  # [S, R, 4] int32: w, h, wA, hA

    def __post_init__(self):
        self.extents = np.ascontiguousarray(self.extents, dtype=np.float64)
        self.volume = np.ascontiguousarray(self.volume, dtype=np.float64)
        S, R = self.extents.shape[0:2]
        dims = np.zeros((S, R, 4), dtype=np.int32)
        for s in range(S):
            assert len(self.tables[s]) == R
            for r in range(R):
                dims[s, r] = window_dims(self.extents[s, r], self.resolutionH, self.resolutionAct)
                for m in self.tables[s][r]:
                    assert m.shape == (dims[s, r, 0], dims[s, r, 1]), (m.shape, dims[s, r])
                    assert m.dtype == np.float64
        self.dims = dims

    @property
    def num_shapes(self):
        return self.extents.shape[0]

    @property
    def num_rotations(self):
        return self.extents.shape[1]

    def shot_info(self):
        """The reference's ``args.shotInfo`` dict (``tools.py:248-279``)."""
        return {s: [tuple(t) for t in self.tables[s]] for s in range(self.num_shapes)}

    @staticmethod
    def from_flat(dims, ext, vol, maps, offsets, resolutionH=0.01, resolutionAct=0.02, name="loaded"):
        """Inverse of ``flat()`` (used to rebuild a library from a fixture or a device upload)."""
        S, R = ext.shape[0:2]
        tables = []
        for s in range(S):
            rows = []
            for r in range(R):
                w, h = int(dims[s, r, 0]), int(dims[s, r, 1])
                o = int(offsets[s, r]); n = w * h
                rows.append(tuple(np.array(maps[o + k * n:o + (k + 1) * n], dtype=np.float64).reshape(w, h)
                                  for k in range(4)))
            tables.append(rows)
        return ShapeLibrary(resolutionH, resolutionAct, np.array(ext), np.array(vol), tables, name=name)

    def flat(self):
        """Flatten for the C-ABI ``irbpp_load_shapes``: returns
        ``(dims int32[S,R,4], ext float64[S,R,3], vol float64[S], maps float64[*],
        offsets int64[S,R])`` with the four maps of (s, r) stored back to back
        ``T | B | mT | mB`` (each ``w*h`` row-major) at ``offsets[s, r]``."""
        S, R = self.num_shapes, self.num_rotations
        offsets = np.zeros((S, R), dtype=np.int64)
        chunks = []
        pos = 0
        for s in range(S):
            for r in range(R):
                offsets[s, r] = pos
                for m in self.tables[s][r]:
                    chunks.append(np.ascontiguousarray(m, dtype=np.float64).ravel())
                    pos += m.size
        maps = np.concatenate(chunks) if chunks else np.zeros(0, dtype=np.float64)
        return self.dims.copy(), self.extents.copy(), self.volume.copy(), maps, offsets


# ---------------------------------------------------------------------------
# the reference's on-disk table cache (tools.shotInfoPre, tools.py:248-279)
# ---------------------------------------------------------------------------

SHOTINFO_META = "irbpp_info.pt"     # not part of the reference layout: extents / volume of a saved library


def shotinfo_dir_name(data_name, dict_name, resolutionH, mesh_scale=1):
    """``dataset/shotInfo/<data>_<dict>_<resH>[_<scale>]`` as ``tools.py:255-260`` composes it."""
    if mesh_scale != 1:
        return "{}_{}_{}_{}".format(data_name, dict_name, resolutionH, mesh_scale)
    return "{}_{}_{}".format(data_name, dict_name, resolutionH)


def save_shotinfo_dir(lib, path):
    """Write ``lib`` in the reference's cache layout: one ``<id>_<rotIdx>.pt`` per (shape, rotation)
    holding ``[heightMapT, heightMapB, maskH, maskB]`` (``tools.py:270-276``; ``torch.save`` of NumPy
    arrays), so that the reference's ``shotInfoPre`` finds and loads them.  Extents and volumes, which
    the reference takes from the meshes (``tools.py:236-241``), go to ``irbpp_info.pt`` beside them."""
    import os
    import torch
    os.makedirs(path, exist_ok=True)
    for s in range(lib.num_shapes):
        for r in range(lib.num_rotations):
            torch.save([np.array(m) for m in lib.tables[s][r]], os.path.join(path, "{}_{}.pt".format(s, r)))
    torch.save({"extents": lib.extents, "volume": lib.volume, "resolutionH": lib.resolutionH,
                "resolutionAct": lib.resolutionAct}, os.path.join(path, SHOTINFO_META))


def load_shotinfo_dir(path, extents=None, volume=None, resolutionH=None, resolutionAct=None, name=None):
    """Read a ``dataset/shotInfo/...`` directory written by the reference's ``shotInfoPre``
    (``tools.py:248-279``) or by ``save_shotinfo_dir`` into a ``ShapeLibrary``.

    The cache holds only the four maps per (id, rotIdx).  ``extents`` ``[S, R, 3]`` (``mesh.extents`` of
    every rotation, ``space.py:104``) and ``volume`` ``[S]`` (``infoDict[id][0]['volume']``,
    ``binPhy.py:151``) come from the caller -- ``args.infoDict`` in the reference -- unless the
    directory carries ``irbpp_info.pt``.  Ids must be ``0..S-1`` with the same rotation count each."""
    import os
    import re
    import torch
    found = {}
    for fn in os.listdir(path):
        m = re.fullmatch(r"(\d+)_(\d+)\.pt", fn)
        if m:
            found[(int(m.group(1)), int(m.group(2)))] = fn
    if not found:
        raise FileNotFoundError("no <id>_<rotIdx>.pt files in %s" % path)
    S = max(k for k, _ in found) + 1
    R = max(r for _, r in found) + 1
    missing = [(k, r) for k in range(S) for r in range(R) if (k, r) not in found]
    if missing:
        raise ValueError("incomplete shotInfo cache, missing %s" % missing[:8])
    meta_path = os.path.join(path, SHOTINFO_META)
    if os.path.exists(meta_path):
        meta = torch.load(meta_path, weights_only=False)
        extents = meta["extents"] if extents is None else extents
        volume = meta["volume"] if volume is None else volume
        resolutionH = meta["resolutionH"] if resolutionH is None else resolutionH
        resolutionAct = meta["resolutionAct"] if resolutionAct is None else resolutionAct
    if extents is None or volume is None or resolutionH is None or resolutionAct is None:
        raise ValueError("extents / volume / resolutions are not in the cache: pass them (args.infoDict, args.resolutionH/A)")
    tables = []
    for k in range(S):
        rows = []
        for r in range(R):
            maps = torch.load(os.path.join(path, found[(k, r)]), weights_only=False)      # tools.py:271
            rows.append(tuple(np.ascontiguousarray(np.asarray(m), dtype=np.float64) for m in maps))
        tables.append(rows)
    return ShapeLibrary(float(resolutionH), float(resolutionAct), np.asarray(extents, dtype=np.float64),
                        np.asarray(volume, dtype=np.float64), tables,
                        name=name or os.path.basename(os.path.normpath(path)))


# ---------------------------------------------------------------------------
# voxel models -> tables (shot_item sampling rule)
# ---------------------------------------------------------------------------

def _voxel_tables(occ, edge, resolutionH, resolutionAct):
    """occ: bool [nx, ny, nz] occupancy with bbox-min at the origin.
    Returns (extents, (T, B, mT, mB))."""
    nx, ny, nz = occ.shape
    extents = np.array([nx * edge, ny * edge, nz * edge], dtype=np.float64)
    w, h, _, _ = window_dims(extents, resolutionH, resolutionAct)
    T = np.zeros((w, h)); B = np.zeros((w, h)); mT = np.zeros((w, h)); mB = np.zeros((w, h))
    for i in range(w):
        x = i * resolutionH + RAY_SHIFT
        cx = int(x // edge)
        if cx >= nx:
            continue
        for j in range(h):
            y = j * resolutionH + RAY_SHIFT
            cy = int(y // edge)
            if cy >= ny:
                continue
            col = np.nonzero(occ[cx, cy])[0]
            if col.size == 0:
                continue
            B[i, j] = col[0] * edge
            T[i, j] = (col[-1] + 1) * edge
            mB[i, j] = 1.0
            mT[i, j] = 1.0
    return extents, (T, B, mT, mB)


def _grow_polycube(rng, n_cells):
    cells = {(0, 0, 0)}
    dirs = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
    cur = (0, 0, 0)
    guard = 0
    while len(cells) < n_cells and guard < 1000:
        guard += 1
        d = dirs[int(rng.integers(0, 6))]
        nxt = (cur[0] + d[0], cur[1] + d[1], cur[2] + d[2])
        cells.add(nxt)
        cur = nxt
    arr = np.array(sorted(cells))
    arr -= arr.min(axis=0)
    occ = np.zeros(arr.max(axis=0) + 1, dtype=bool)
    occ[arr[:, 0], arr[:, 1], arr[:, 2]] = True
    return occ


def make_blockout_library(num_shapes=32, seed=1, num_rotations=4, edge=0.04,
                          resolutionH=0.01, resolutionAct=0.02, min_cells=2, max_cells=5):
    """BlockOut-like polycubes (SURVEY.md 8d): ``n in [min_cells, max_cells]`` cells grown by a
    random face-adjacent walk, rotations = rot90 about z."""
    rng = np.random.default_rng(seed)
    ext = np.zeros((num_shapes, num_rotations, 3)); vol = np.zeros(num_shapes); tables = []
    for s in range(num_shapes):
        occ = _grow_polycube(rng, int(rng.integers(min_cells, max_cells + 1)))
        vol[s] = occ.sum() * edge ** 3
        rows = []
        for r in range(num_rotations):
            occ_r = np.rot90(occ, k=r, axes=(0, 1))
            e, t = _voxel_tables(occ_r, edge, resolutionH, resolutionAct)
            ext[s, r] = e
            rows.append(t)
        tables.append(rows)
    return ShapeLibrary(resolutionH, resolutionAct, ext, vol, tables, name="blockout_synth")


def make_cube_library(seed=1, num_rotations=2, resolutionH=0.01, resolutionAct=0.02,
                      edges=(0.03, 0.06, 0.09, 0.12, 0.15), num_shapes=None):
    """Cube-dataset stand-in: boxes with edges from ``edges`` (reference README.md:39), R = 2."""
    rng = np.random.default_rng(seed)
    combos = [(a, b, c) for a in edges for b in edges for c in edges]
    if num_shapes is not None:
        idx = rng.permutation(len(combos))[:num_shapes]
        combos = [combos[i] for i in sorted(idx)]
    S = len(combos)
    ext = np.zeros((S, num_rotations, 3)); vol = np.zeros(S); tables = []
    for s, (a, b, c) in enumerate(combos):
        vol[s] = a * b * c
        rows = []
        for r in range(num_rotations):
            e = np.array([a, b, c]) if r % 2 == 0 else np.array([b, a, c])
            w, h, _, _ = window_dims(e, resolutionH, resolutionAct)
            T = np.zeros((w, h)); B = np.zeros((w, h)); mT = np.zeros((w, h)); mB = np.zeros((w, h))
            xs = np.arange(w) * resolutionH + RAY_SHIFT
            ys = np.arange(h) * resolutionH + RAY_SHIFT
            hit = (xs[:, None] < np.round(e[0], 6)) & (ys[None, :] < np.round(e[1], 6))
            T[hit] = e[2]; mT[hit] = 1.0; mB[hit] = 1.0
            ext[s, r] = e
            rows.append((T, B, mT, mB))
        tables.append(rows)
    return ShapeLibrary(resolutionH, resolutionAct, ext, vol, tables, name="cube_synth")


def _irregular_field(rng, ex, ey, ez, resolutionH, resolutionAct, lift_bottom):
    e = np.array([ex, ey, ez], dtype=np.float64)
    w, h, _, _ = window_dims(e, resolutionH, resolutionAct)
    xs = np.arange(w) * resolutionH + RAY_SHIFT
    ys = np.arange(h) * resolutionH + RAY_SHIFT
    inside = (xs[:, None] < np.round(ex, 6)) & (ys[None, :] < np.round(ey, 6))
    # footprint: union of a few ellipses, minus an optional hole
    X, Y = np.meshgrid(xs / ex, ys / ey, indexing="ij")
    foot = np.zeros((w, h), dtype=bool)
    for _ in range(int(rng.integers(1, 4))):
        cx, cy = rng.uniform(0.25, 0.75, size=2)
        ax, ay = rng.uniform(0.2, 0.6, size=2)
        foot |= ((X - cx) / ax) ** 2 + ((Y - cy) / ay) ** 2 <= 1.0
    if rng.random() < 0.4:
        cx, cy = rng.uniform(0.3, 0.7, size=2)
        foot &= ~(((X - cx) / 0.15) ** 2 + ((Y - cy) / 0.15) ** 2 <= 1.0)
    foot &= inside
    if not foot.any():
        foot = inside.copy()
    # smooth bottom and top surfaces (metres, arbitrary float64 values)
    gx, gy = rng.uniform(-1, 1, size=2)
    bowl = rng.uniform(0, 1)
    bottom = 0.35 * ez * (gx * (X - 0.5) + gy * (Y - 0.5) + bowl * ((X - 0.5) ** 2 + (Y - 0.5) ** 2))
    bottom = bottom - bottom[foot].min()
    if lift_bottom:  # every sampled ray hits above the bbox floor (posZ can go negative)
        bottom = bottom + 0.07 * ez
    bottom = np.minimum(bottom, 0.6 * ez)
    tx, ty = rng.uniform(-1, 1, size=2)
    top = ez * (1.0 - 0.25 * np.abs(tx * (X - 0.5) + ty * (Y - 0.5)))
    top = top * (ez / top[foot].max())
    top = np.maximum(top, bottom + 0.1 * ez)
    top = np.minimum(top, ez)
    T = np.where(foot, top, 0.0); B = np.where(foot, bottom, 0.0)
    m = foot.astype(np.float64)
    vol = float(((T - B) * m).sum() * resolutionH * resolutionH)
    return e, (T, B, m.copy(), m.copy()), vol


def make_irregular_library(num_shapes=32, seed=1, num_rotations=8, resolutionH=0.01, resolutionAct=0.02,
                           lift_fraction=0.15):
    """General / Kitchen / ABC stand-in (SURVEY.md 8d): irregular height fields with non-flat
    bottoms, holes in the masks and extents that are not multiples of the resolutions, so the
    ``ceil`` / ``round`` hazards of ``space.py:104-106`` are exercised.  Rotation r>0 is the rot90
    family of two independent fields (the second stands for the 45-degree pose with a larger
    bounding box), which is all the environment can observe of a rotation."""
    rng = np.random.default_rng(seed)
    ext = np.zeros((num_shapes, num_rotations, 3)); vol = np.zeros(num_shapes); tables = []
    for s in range(num_shapes):
        ex, ey = rng.uniform(0.03, 0.15, size=2)
        ez = rng.uniform(0.02, 0.12)
        if rng.random() < 0.3:  # snap some extents to grid multiples (float-noise hazards)
            ex = round(ex / 0.01) * 0.01
            ey = round(ey / 0.02) * 0.02
        lift = rng.random() < lift_fraction
        base = [_irregular_field(rng, ex, ey, ez, resolutionH, resolutionAct, lift)]
        grow = float(rng.uniform(1.05, 1.35))
        base.append(_irregular_field(rng, min(ex * grow, 0.2), min(ey * grow, 0.2), ez,
                                     resolutionH, resolutionAct, lift))
        vol[s] = base[0][2]
        rows = []
        for r in range(num_rotations):
            e, (T, B, mT, mB), _ = base[(r // 4) % 2]
            k = r % 4
            e_r = np.array([e[0], e[1], e[2]]) if k % 2 == 0 else np.array([e[1], e[0], e[2]])
            w, h, _, _ = window_dims(e_r, resolutionH, resolutionAct)
            maps = []
            for m in (T, B, mT, mB):
                mr = np.ascontiguousarray(np.rot90(m, k=k))
                out = np.zeros((w, h))
                out[:min(w, mr.shape[0]), :min(h, mr.shape[1])] = mr[:w, :h]
                maps.append(out)
            ext[s, r] = e_r
            rows.append(tuple(maps))
        tables.append(rows)
    return ShapeLibrary(resolutionH, resolutionAct, ext, vol, tables, name="irregular_synth")


def make_sequences(num_envs, length, num_shapes, seed=0):
    """Per-env item-id sequences ``ids[N, L]`` (SURVEY.md 8d): i.i.d. uniform ids from
    ``np.random.default_rng(seed + env)`` -- the stand-in for ``RandomItemCreator``
    (reference ``IRcreator.py:26-33``) so that both sides see identical shape sequences."""
    out = np.zeros((num_envs, length), dtype=np.int32)
    for e in range(num_envs):
        out[e] = np.random.default_rng(seed + e).integers(0, num_shapes, size=length)
    return out


def item_rng_ids(seed, num_envs, count, num_shapes):
    """The ids the device draws in item-generator mode (``irbpp_set_item_rng``): env e's d-th draw is
    ``mix(seed, e, d) mod num_shapes`` with the splitmix64 finaliser of ``csrc/irbpp_kernels.cuh``
    (``item_rng``).  Returns ``ids[num_envs, count]`` int32 -- used by the tests to give the CPU oracle
    the very same i.i.d. stream (the stand-in for ``RandomItemCreator``, reference ``IRcreator.py:26-33``)."""
    z = _splitmix64(seed, num_envs, count)
    return ((z >> np.uint64(32)) % np.uint64(num_shapes)).astype(np.int32)


def _splitmix64(seed, num_envs, count):
    """``splitmix64(seed, e, d)`` of ``csrc/irbpp_kernels.cuh`` for every env e and draw d: uint64 [num_envs, count]."""
    M = np.uint64(0xFFFFFFFFFFFFFFFF)
    e = np.arange(num_envs, dtype=np.uint64)[:, None]
    d = np.arange(count, dtype=np.uint64)[None, :]
    g = np.uint64(0x9E3779B97F4A7C15)
    with np.errstate(over="ignore"):
        z = (np.uint64(seed) + g * ((e << np.uint64(32)) | d) + g) & M
        z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & M
        z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & M
        return z ^ (z >> np.uint64(31))


def instance_groups(id2shape):
    """The groups ``RandomInstanceCreator`` draws from (reference ``IRcreator.py:35-50``): the ids of the id -> file
    dict (``args.dicPath``) keyed by ``name[0:-6]`` -- the file name without its pose suffix -- in the order the dict
    lists them.  Returns a list of id lists."""
    inverse = {}
    for k, name in id2shape.items():
        inverse.setdefault(name[0:-6], []).append(k)
    return list(inverse.values())


CATEGORIES = ("objects", "concave", "board")     # IRcreator.py:55; the declared weights are never used


def category_groups(id2shape):
    """The groups ``RandomCateCreator`` draws from (reference ``IRcreator.py:52-72``): the ids of each of the fixed
    categories ``objects / concave / board``, by the ``category/file`` prefix of their name; the category is chosen
    uniformly.  An empty category raises ``ValueError`` (the reference would fail at its first draw)."""
    cates = {c: [] for c in CATEGORIES}
    for k, name in id2shape.items():
        cate, _ = name.split("/")
        if cate not in cates:
            raise ValueError("unknown category %r of item %r" % (cate, k))
        cates[cate].append(k)
    for c, ids in cates.items():
        if not ids:
            raise ValueError("category %r has no item" % c)
    return list(cates.values())


def group_table(groups):
    """Groups (lists of ids) -> the CSR form of ``irbpp_set_item_groups``: ``(offsets int32[G + 1], members int32)``."""
    sizes = [len(g) for g in groups]
    offsets = np.zeros(len(groups) + 1, dtype=np.int32)
    offsets[1:] = np.cumsum(sizes)
    members = np.array([int(i) for g in groups for i in g], dtype=np.int32)
    return offsets, members


def item_group_ids(seed, num_envs, count, groups):
    """The ids the device draws with item groups (``irbpp_set_item_groups``): env e's d-th draw takes
    ``z = splitmix64(seed, e, d)``, group ``hi32(z) mod G`` and member ``lo32(z) mod n_g`` of it.  Returns
    ``ids[num_envs, count]`` int32 -- the Python mirror of the device stream."""
    offsets, members = group_table(groups)
    z = _splitmix64(seed, num_envs, count)
    g = ((z >> np.uint64(32)) % np.uint64(len(groups))).astype(np.int64)
    lo = z & np.uint64(0xFFFFFFFF)
    n = (offsets[g + 1] - offsets[g]).astype(np.uint64)
    return members[offsets[g] + (lo % n).astype(np.int64)].astype(np.int32)


def load_trajectories(path_or_list):
    """Item trajectories as ``LoadItemCreator`` reads them (reference ``IRcreator.py:74-80``): ``test_sequence.pt`` is
    a ``torch.load``-ed list of id lists.  Accepts that path or the list itself; returns a list of int lists (a copy:
    the reference's creator appends ``None`` to the lists it plays)."""
    trajs = path_or_list
    if isinstance(path_or_list, (str, bytes)) or hasattr(path_or_list, "__fspath__"):
        import torch
        trajs = torch.load(path_or_list, weights_only=False)
    return [[int(i) for i in t] for t in trajs]


def trajectory_table(trajectories):
    """Trajectories -> the ragged form of ``irbpp_set_trajectories``: ``(items int32, offsets int64[T + 1])``."""
    offsets = np.zeros(len(trajectories) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(t) for t in trajectories])
    items = np.array([int(i) for t in trajectories for i in t], dtype=np.int32)
    return items, offsets
