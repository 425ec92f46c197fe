"""``make_vec_envs`` mirror (reference ``envs.py:67-99``).

The reference builds ``VecPyTorch(ShmemVecEnv([make_env(...)] * num_processes))`` from an argparse
namespace that carries the datasets.  Here the same call returns a ``GpuVecEnv`` with the same triple
``(envs, [observation_space, action_space], obs_len)``.  ``args`` needs only the attributes the hot
path reads (``binPhy.py:25-49``):

    num_processes, device, bin_dimension, resolutionA, resolutionH, resolutionZ, ZRotNum,
    selectedAction, bufferSize, seed

plus the shape data: ``args.shapeLibrary`` (a ``shapes.ShapeLibrary``) or the reference's own
``args.shotInfo`` / ``args.shapeDict`` (extents) / ``args.infoDict`` (volumes), and optionally
``args.itemSequences`` (int ids ``[num_processes, L]``, replayed modulo L).  Without it the ids are drawn ON THE
DEVICE, seeded with ``args.seed``, as the reference's ``args.dataSample`` selects (``binPhy.py:58-67``): 'instance' /
'category' draw a group uniformly, then an id within it, from the groups of the id -> file dict ``args.dicPath``
(``RandomInstanceCreator`` / ``RandomCateCreator``, ``IRcreator.py:35-72``); 'pose' or no ``dataSample`` draws
i.i.d. uniform ids (``RandomItemCreator``, ``IRcreator.py:26-33``).  Neither has a period.  ``args.approxLegacy`` (optional, default
False) selects the older point-to-line ``approxPolyDP`` rule (the reference pins OpenCV 4.4.0.46)."""
import numpy as np

from . import shapes
from .vec_env import GpuVecEnv


def library_from_reference_args(args):
    """Build a ``ShapeLibrary`` from the reference's ``shotInfo`` / ``shapeDict`` / ``infoDict``."""
    shot = args.shotInfo
    ids = sorted(shot.keys())
    R = len(shot[ids[0]])
    ext = np.zeros((len(ids), R, 3)); vol = np.zeros(len(ids)); tables = []
    for s, k in enumerate(ids):
        for r in range(R):
            ext[s, r] = np.asarray(args.shapeDict[k][r].extents, dtype=np.float64)   # space.py:104
        vol[s] = float(args.infoDict[k][0]["volume"])                                   # binPhy.py:151
        tables.append([tuple(np.asarray(m, dtype=np.float64) for m in shot[k][r]) for r in range(R)])
    return shapes.ShapeLibrary(args.resolutionH, args.resolutionA, ext, vol, tables, name="reference_args")


def make_vec_envs(args, log_dir=None, allow_early_resets=True):
    """-> ``(envs, [observation_space, action_space], obs_len)`` as reference ``envs.py:67-99``.
    ``log_dir`` / ``allow_early_resets`` are accepted for signature compatibility (the Monitor CSV of
    ``envs.py:48-52`` is not written; episode info is delivered in ``infos`` as the trainer reads it)."""
    lib = getattr(args, "shapeLibrary", None)
    if lib is None:
        lib = library_from_reference_args(args)
    n = int(args.num_processes)
    seqs = getattr(args, "itemSequences", None)
    groups = None
    if seqs is None:
        groups = item_groups_from_args(args)           # None: i.i.d. uniform ids generated on the device
    envs = GpuVecEnv(lib, seqs, num_envs=n, device=getattr(args, "device", "cuda:0"), item_groups=groups,
                     item_seed=int(getattr(args, "seed", 0)), **_env_kwargs(args))
    return envs, [envs.observation_space, envs.action_space], envs.obs_len


def _env_kwargs(args):
    return dict(approx_legacy=bool(getattr(args, "approxLegacy", False)),
                selected_action=int(getattr(args, "selectedAction", 500)),
                buffer_size=int(getattr(args, "bufferSize", 1)),
                bin_dimension=tuple(getattr(args, "bin_dimension", (0.32, 0.32, 0.30))),
                resolution_act=float(getattr(args, "resolutionA", 0.02)),
                resolution_h=float(getattr(args, "resolutionH", 0.01)),
                resolution_z=float(getattr(args, "resolutionZ", 0.01)))


def item_groups_from_args(args):
    """The groups ``binPhy.py:58-67`` builds its item creator from: ``args.dataSample`` 'instance' ->
    ``shapes.instance_groups``, 'category' -> ``shapes.category_groups`` of the id -> file dict ``args.dicPath`` (a
    path loaded with ``torch.load``, or the dict itself); 'pose' or no ``dataSample``: None (uniform ids)."""
    sample = getattr(args, "dataSample", None)
    if sample in (None, "pose"):
        return None
    if sample not in ("instance", "category"):
        raise ValueError("unknown dataSample %r" % (sample,))
    d = args.dicPath
    if not isinstance(d, dict):
        import torch
        d = torch.load(d, weights_only=False)
    return shapes.instance_groups(d) if sample == "instance" else shapes.category_groups(d)


def make_eval_env(args):
    """``make_eval_env`` (reference ``tools.py:433``): one bin that plays the trajectories of ``args.test_name`` (a
    ``test_sequence.pt`` path, or the list itself) from trajectory 1 on, as ``LoadItemCreator`` does under
    ``tools.test``."""
    from .single_env import SingleGpuEnv
    lib = getattr(args, "shapeLibrary", None)
    if lib is None:
        lib = library_from_reference_args(args)
    return SingleGpuEnv(lib, trajectories=shapes.load_trajectories(args.test_name), first_trajectory=1,
                        device=getattr(args, "device", "cuda:0"), **_env_kwargs(args))
