"""DQNBPP's height encoder on the device (``csrc/irbpp_height_encoder.cuh``), forward and backward, as a drop-in module.

The reference's ``heightEncoder`` (``model.py:258-264``) is the same ``nn.Sequential`` at both network levels: three
convolutions, each followed by LeakyReLU.  Trained with cudnn off, as the reference trains by default, torch runs each
convolution and its backward pass one sample at a time.  ``DeviceHeightEncoder`` keeps the module's children, so its
parameters, ``state_dict`` keys and optimiser state stay what they were, and runs ``forward`` and the backward pass
as kernels, one CTA per sample::

    agent.online_net.heightEncoder = DeviceHeightEncoder(agent.online_net.heightEncoder)
    agent.target_net.heightEncoder = DeviceHeightEncoder(agent.target_net.heightEncoder)

Autograd reaches the kernels through a ``torch.autograd.Function`` whose inputs are the heightmap and the six conv
tensors; its backward pass returns the six weight gradients, summed over the batch in a fixed order (two calls give
bit-identical results), and no gradient for the heightmap, which is an observation.  Double backward is not supported.
There is no CPU path: a CPU input raises ``ValueError``."""
import ctypes
import math

import torch
from torch import nn

from . import _lib

HM = 32
# child name -> (in_channels, out_channels, kernel, stride, padding) of the reference's convolutions
CONVS = (("conv1", (1, 16, 4, 2, 1)), ("conv2", (16, 32, 4, 2, 1)), ("conv3", (32, 4, 3, 1, 1)))
RELUS = ("relu1", "relu2", "relu3")
CHILDREN = ("conv1", "relu1", "conv2", "relu2", "conv3", "relu3")
STRUCTURE = ("conv1 Conv2d(1, 16, 4, stride 2, padding 1), relu1 LeakyReLU, conv2 Conv2d(16, 32, 4, stride 2, padding 1), "
             "relu2 LeakyReLU, conv3 Conv2d(32, 4, 3, stride 1, padding 1), relu3 LeakyReLU, one slope >= 0")


def _slope_of(modules):
    """The LeakyReLU slope the three activations share; ``ValueError`` unless it is one finite value >= 0."""
    slopes = set(float(modules[n].negative_slope) for n in RELUS)
    if len(slopes) != 1:
        raise ValueError("the three LeakyReLU have different slopes %s; supported: %s" % (sorted(slopes), STRUCTURE))
    slope = slopes.pop()
    if not (math.isfinite(slope) and slope >= 0.0):
        raise ValueError("LeakyReLU slope %r is not a finite value >= 0; supported: %s" % (slope, STRUCTURE))
    return slope


def _check_structure(seq):
    if not isinstance(seq, nn.Sequential):
        raise ValueError("expected the heightEncoder nn.Sequential, got %s" % type(seq).__name__)
    names = tuple(n for n, _ in seq.named_children())
    if names != CHILDREN:
        raise ValueError("heightEncoder has the children %s; supported: %s" % (list(names), STRUCTURE))
    mods = dict(seq.named_children())
    for name, (cin, cout, k, s, p) in CONVS:
        m = mods[name]
        if not isinstance(m, nn.Conv2d):
            raise ValueError("%s is a %s, not Conv2d; supported: %s" % (name, type(m).__name__, STRUCTURE))
        got = (m.in_channels, m.out_channels, tuple(m.kernel_size), tuple(m.stride), tuple(m.padding),
               tuple(m.dilation), m.groups, m.bias is not None, m.padding_mode)
        if got != (cin, cout, (k, k), (s, s), (p, p), (1, 1), 1, True, "zeros"):
            raise ValueError("%s is %s; supported: %s" % (name, m, STRUCTURE))
    for name in RELUS:
        if not isinstance(mods[name], nn.LeakyReLU):
            raise ValueError("%s is a %s, not LeakyReLU; supported: %s" % (name, type(mods[name]).__name__, STRUCTURE))
    return _slope_of(mods)


class DeviceHeightEncoder(nn.Sequential):
    """``seq`` (a reference ``heightEncoder``) with the same child modules under the same names; ``forward`` runs
    ``irbpp_height_encoder_forward`` and its backward pass ``irbpp_height_encoder_backward``.  Input: float32 CUDA
    ``[B, 1, 32, 32]`` heightmaps, B >= 1, not requiring grad (a view into observation rows is read in place); output
    ``[B, 4, 8, 8]`` as the Sequential returns it."""

    def __init__(self, seq):
        _check_structure(seq)
        super().__init__()
        for name, m in seq.named_children():
            self.add_module(name, m)
        self.train(seq.training)

    def _weights(self, device):
        ws = []
        for name, _ in CONVS:
            conv = getattr(self, name)
            for t in (conv.weight, conv.bias):
                if t.device != device:
                    raise ValueError("heightEncoder weights live on %s, the input on %s" % (t.device, device))
                if t.dtype != torch.float32:
                    raise ValueError("heightEncoder weights must be float32, got %s" % t.dtype)
                ws.append(t.contiguous())
        return ws

    def forward(self, hm):
        if not isinstance(hm, torch.Tensor) or not hm.is_cuda:
            raise ValueError("the heightmap must be a CUDA tensor [B, 1, %d, %d] (there is no CPU path)" % (HM, HM))
        if hm.dtype != torch.float32:
            raise ValueError("the heightmap must be float32, got %s" % hm.dtype)
        if hm.dim() != 4 or tuple(hm.shape[1:]) != (1, HM, HM) or hm.shape[0] < 1:
            raise ValueError("the heightmap must be [B >= 1, 1, %d, %d], got %s" % (HM, HM, tuple(hm.shape)))
        if hm.requires_grad:
            raise ValueError("the heightmap requires grad; it is an observation and gets no gradient")
        slope = _slope_of(dict(self.named_children()))
        ws = self._weights(hm.device)
        # sample b's 1024 values must be contiguous at hm + b * stride(0) with stride(0) >= 1024
        if hm.stride(3) != 1 or hm.stride(2) != HM or hm.stride(0) < HM * HM:
            hm = hm.contiguous()
        return _HeightEncoderFunction.apply(hm, slope, *ws)


def _weights_struct(ws, slope):
    return _lib.IrbppHeightEncoderWeights(*([t.data_ptr() for t in ws] + [ctypes.c_float(slope)]))


class _HeightEncoderFunction(torch.autograd.Function):
    """The heightmap and the six conv tensors in, the map ``[B, 4, 8, 8]`` out; the backward pass returns the six
    weight gradients and none for the heightmap or the slope."""

    @staticmethod
    def forward(ctx, hm, slope, *ws):
        lib = _lib.load()
        B = hm.shape[0]
        w = _weights_struct(ws, slope)
        out = torch.empty((B, 4, 8, 8), dtype=torch.float32, device=hm.device)
        rc = lib.irbpp_height_encoder_forward(ctypes.byref(w), hm.data_ptr(), hm.stride(0), B, out.data_ptr(),
                                              torch.cuda.current_stream(hm.device).cuda_stream)
        _lib.check(lib, None, rc)
        ctx.slope = slope
        ctx.save_for_backward(hm, *ws)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad):
        lib = _lib.load()
        hm, ws = ctx.saved_tensors[0], ctx.saved_tensors[1:]
        B, dev = hm.shape[0], hm.device
        grad = grad.to(torch.float32).contiguous()
        w = _weights_struct(ws, ctx.slope)
        dws = [torch.empty(t.shape, dtype=torch.float32, device=dev) for t in ws]
        g = _lib.IrbppHeightEncoderGrads(*[t.data_ptr() for t in dws])
        nbytes = int(lib.irbpp_height_encoder_scratch_bytes(B))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)        # the caching allocator aligns to 512 bytes
        rc = lib.irbpp_height_encoder_backward(ctypes.byref(w), hm.data_ptr(), hm.stride(0), B, grad.data_ptr(),
                                               ctypes.byref(g), scratch.data_ptr(), nbytes,
                                               torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(lib, None, rc)
        return (None, None) + tuple(dws)
