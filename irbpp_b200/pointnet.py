"""The next item's point-cloud feature on the device (SURVEY.md 8(f)3).

Reference ``model.py:328-335`` (location level) and ``:366-372`` (order level)::

    nextShape = self.shapeArray[next_item_ID.cpu()]                       # HOST gather, [B, 100000, 3] rows
    indices   = np.random.randint(self.shapeArray.shape[1], size=self.args.samplePointsNum)
    nextShape = nextShape[:, indices].to(self.args.device)               # H2D of [B, 1024, 3] every forward
    shape_feature = torch.max(self.shapeEncoder(nextShape), dim=1)[0]    # Linear(3,128) LeakyReLU Linear(128,128) LeakyReLU

``DeviceShapeClouds`` keeps ``shapeArray`` resident on the GPU and serves both forms through the C ABI
(``include/irbpp.h``): ``sample`` returns the reference's ``nextShape`` tensor (drop-in: the caller keeps its
encoder), ``features`` returns ``shape_feature`` directly -- the encoder evaluated once per library SHAPE (the
index set is shared by the batch, so the feature depends on the shape only) and gathered per bin.  One index set
per forward pass comes from a counter-based generator (``pn_indices`` mirrors it on the host); float32.
"""
import ctypes

import numpy as np

from . import _lib

PN_H = 128


def pn_indices(seed, counter, n_points, num_cloud_points):
    """Host mirror of the device index generator (``csrc/irbpp_pointnet.cuh`` ``pn_index``): the index set of
    forward pass ``counter`` -- uniform with replacement over the cloud, the role of ``np.random.randint``."""
    M = np.uint64(0xFFFFFFFFFFFFFFFF)
    j = np.arange(n_points, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * (((np.uint64(counter) << np.uint64(20)) & M) ^ j)
             + np.uint64(0xD1B54A32D192ED03)) & M
        z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & M
        z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & M
        z = z ^ (z >> np.uint64(31))
    return ((z >> np.uint64(32)) % np.uint64(num_cloud_points)).astype(np.int64)


class DeviceShapeClouds(object):
    """``shapeArray`` (``[S, P, 3]`` float32, ``tools.shapeProcessing``, reference ``tools.py:211-225``) resident on
    one GPU.  ``item_col`` is where the observation carries the next item id (``selectedAction * 5``,
    ``binPhy.py:191,227``)."""

    def __init__(self, shape_array, device="cuda:0", n_points=1024, seed=0, item_col=2500):
        import torch
        self._torch = torch
        self._lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("DeviceShapeClouds needs a CUDA device; there is no CPU path")
        arr = torch.as_tensor(np.asarray(shape_array, dtype=np.float32)) if not isinstance(shape_array, torch.Tensor) else shape_array
        if arr.dim() != 3 or arr.shape[2] != 3:
            raise ValueError("shape_array must be [S, P, 3]")
        self.shape_array = arr.to(self.device, torch.float32).contiguous()
        self.S, self.P = int(arr.shape[0]), int(arr.shape[1])
        self.n_points, self.seed, self.item_col = int(n_points), int(seed), int(item_col)
        self.counter = 0                       # forward passes served so far (one index set each)
        self._keys = torch.empty(self.S * PN_H, dtype=torch.int32, device=self.device)

    def _stream(self):
        return self._torch.cuda.current_stream(self.device).cuda_stream

    def _item_args(self, obs_or_ids):
        torch = self._torch
        t = obs_or_ids
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError("expected a CUDA tensor: the observations [B, obs_len] or int item ids [B]")
        if t.device != self.device:
            raise ValueError("observations live on %s, the point clouds on %s" % (t.device, self.device))
        if t.dtype in (torch.int32, torch.int64):
            ids = t.reshape(-1).to(torch.int32).contiguous()
            return ids, 0, 0, 0, ids.data_ptr(), ids.numel()
        obs = t.contiguous() if t.stride(-1) != 1 else t
        return obs, obs.data_ptr(), obs.stride(0), self.item_col, 0, obs.shape[0]

    def _check(self, rc):
        if rc != _lib.IRBPP_OK:
            msg = self._lib.irbpp_last_error(None)
            raise _lib.IrbppError(rc, msg.decode() if msg else "?")

    def sample(self, obs_or_ids, counter=None, return_indices=False):
        """``nextShape`` of model.py:330-332: float32 ``[B, n_points, 3]`` on the device."""
        torch = self._torch
        keep, obs_ptr, stride, col, ids_ptr, B = self._item_args(obs_or_ids)
        c = self.counter if counter is None else int(counter)
        out = torch.empty((B, self.n_points, 3), dtype=torch.float32, device=self.device)
        idx = torch.empty(self.n_points, dtype=torch.int32, device=self.device) if return_indices else None
        self._check(self._lib.irbpp_sample_point_clouds(self.shape_array.data_ptr(), self.S, self.P, obs_ptr, stride, col, ids_ptr,
                                                        B, self.seed, c, self.n_points, out.data_ptr(),
                                                        idx.data_ptr() if idx is not None else 0, self._stream()))
        if counter is None:
            self.counter += 1
        return (out, idx) if return_indices else out

    def features(self, obs_or_ids, encoder, counter=None):
        """``shape_feature`` of model.py:334-335: float32 ``[B, 128]``.  ``encoder`` is the reference's
        ``shapeEncoder`` (an ``nn.Sequential`` with ``linear1`` / ``linear2`` and LeakyReLU) or a tuple
        ``(W1 [128,3], b1 [128], W2 [128,128], b2 [128], negative_slope)`` of CUDA float32 tensors."""
        torch = self._torch
        if isinstance(encoder, tuple):
            W1, b1, W2, b2, slope = encoder
        else:
            mods = list(encoder.children())
            lin = [m for m in mods if hasattr(m, "weight")]
            act = [m for m in mods if hasattr(m, "negative_slope")]
            W1, b1, W2, b2 = lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias
            slope = float(act[0].negative_slope) if act else 0.01
        ws = [w.detach().to(self.device, torch.float32).contiguous() for w in (W1, b1, W2, b2)]
        if tuple(ws[0].shape) != (PN_H, 3) or tuple(ws[2].shape) != (PN_H, PN_H):
            raise ValueError("shapeEncoder must be Linear(3,128) -> Linear(128,128) (model.py:266-270)")
        keep, obs_ptr, stride, col, ids_ptr, B = self._item_args(obs_or_ids)
        c = self.counter if counter is None else int(counter)
        out = torch.empty((B, PN_H), dtype=torch.float32, device=self.device)
        self._check(self._lib.irbpp_shape_features(self.shape_array.data_ptr(), self.S, self.P, obs_ptr, stride, col, ids_ptr, B,
                                                   self.seed, c, self.n_points, ws[0].data_ptr(), ws[1].data_ptr(),
                                                   ws[2].data_ptr(), ws[3].data_ptr(), ctypes.c_float(slope),
                                                   self._keys.data_ptr(), out.data_ptr(), self._stream()))
        if counter is None:
            self.counter += 1
        return out


# ---- the order level's point rule (model.py:240-244, 301-306, 365-368, 401-403) ----
ORDER_ARRAY_POINTS = 10000          # arrayPointNum: the points of each shape's subsample
ORDER_REDRAW = 1000                 # the subsample is redrawn every 1000 forward passes
_SUBSAMPLE_STREAM = 1 << 40         # generator counters of the subsamples, apart from those of the acts (< 2**40)


def order_point_indices(seed, act, n_points, num_cloud_points):
    """Host mirror of ``OrderShapeClouds``: the cloud points (indices into ``shapeArray``'s second axis) of act
    ``act``, the act's draw mapped through the subsample of its epoch ``act // 1000``."""
    sub = pn_indices(seed, _SUBSAMPLE_STREAM + act // ORDER_REDRAW, ORDER_ARRAY_POINTS,
                     min(num_cloud_points, ORDER_ARRAY_POINTS))
    return sub[pn_indices(seed, act, n_points, ORDER_ARRAY_POINTS)]


class OrderShapeClouds(object):
    """The order network's point rule over a ``DeviceShapeClouds`` (opt-in; the default path samples the whole cloud).

    The reference's order level keeps a subsample of 10 000 points per shape, drawn with replacement from the first
    10 000 points of each cloud (``np.random.randint(self.shapeArray.shape[1])`` there reads the subsample's own
    size) and redrawn every 1000 forward passes; each forward draws ``samplePointsNum`` of those 10 000.  Here both
    draws come from the counter-based generator of ``DeviceShapeClouds`` (``order_point_indices`` mirrors them on the
    host).  A cloud of fewer than 10 000 points is subsampled over all its points (the reference raises there)."""

    def __init__(self, clouds):
        self.clouds = clouds
        self.S, self.device, self.item_col = clouds.S, clouds.device, clouds.item_col
        self.counter = 0                    # acts served so far
        self._epoch, self._sub = None, None

    def _subsample(self, c):
        """The ``DeviceShapeClouds`` of act ``c``'s subsample epoch (redrawn when the epoch changes)."""
        torch = self.clouds._torch
        epoch = c // ORDER_REDRAW
        if epoch != self._epoch:
            src = self.clouds
            idx = pn_indices(src.seed, _SUBSAMPLE_STREAM + epoch, ORDER_ARRAY_POINTS, min(src.P, ORDER_ARRAY_POINTS))
            self._sub = DeviceShapeClouds(src.shape_array[:, torch.as_tensor(idx, device=src.device)], device=src.device,
                                          n_points=src.n_points, seed=src.seed, item_col=src.item_col)
            self._epoch = epoch
        return self._sub

    def features(self, obs_or_ids, encoder, counter=None):
        """``DeviceShapeClouds.features`` on the current subsample: float32 ``[B, 128]``."""
        c = self.counter if counter is None else int(counter)
        out = self._subsample(c).features(obs_or_ids, encoder, counter=c)
        if counter is None:
            self.counter += 1
        return out

    def sample(self, obs_or_ids, counter=None):
        """``DeviceShapeClouds.sample`` on the current subsample: float32 ``[B, n_points, 3]``, exactly the points
        ``features`` encodes for the same counter (``order_point_indices``), so that a module's own shape encoder can
        be trained on them."""
        c = self.counter if counter is None else int(counter)
        out = self._subsample(c).sample(obs_or_ids, counter=c)
        if counter is None:
            self.counter += 1
        return out
