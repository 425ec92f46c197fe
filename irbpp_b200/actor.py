"""The location network's forward pass and ``Agent.act`` for every bin on the device (``csrc/irbpp_actor.cuh``).

Reference ``Agent.act`` (``agent.py:51-58``) runs ``DQNBPP.forward`` (``model.py:316-352, 386-404``, location level)
on ``[N, obs_len]`` observations, takes the expected value over the support, masks and takes the argmax over the
``selectedAction`` candidate rows.  ``DeviceActor`` does the same in two kernel launches (plus the shape-feature
launches of ``DeviceShapeClouds.features``), reading the network's weights by the reference's ``state_dict`` keys::

    actor = DeviceActor(agent.online_net, clouds, agent.support)
    action = actor.act(state, mask)                # drop-in for agent.act(state, mask)

A live module is read at every call (weights change after every ``learn`` and ``reset_noise``); its ``training`` flag
selects NoisyLinear's mode (train: ``mu + sigma * epsilon``, eval: ``mu``), built with the reference's own torch
expression on the device.  A plain state dict (``Agent.save`` / ``torch.save(net.state_dict())``) is copied to the
device once and takes the mode from ``train=``.
"""
import ctypes

from . import _lib

HM = 32
EMB = 128
MAX_ATOMS = 32
NOISY = ("fc_h_v", "fc_z_v", "fc_h_a", "fc_z_a")
# key -> shape (None: the number of atoms)
PLAIN_SHAPES = {
    "heightEncoder.conv1.weight": (16, 1, 4, 4), "heightEncoder.conv1.bias": (16,),
    "heightEncoder.conv2.weight": (32, 16, 4, 4), "heightEncoder.conv2.bias": (32,),
    "heightEncoder.conv3.weight": (4, 32, 3, 3), "heightEncoder.conv3.bias": (4,),
    "shapeEncoder.linear1.weight": (EMB, 3), "shapeEncoder.linear1.bias": (EMB,),
    "shapeEncoder.linear2.weight": (EMB, EMB), "shapeEncoder.linear2.bias": (EMB,),
    "init_candidate_embed.0.weight": (32, 4), "init_candidate_embed.0.bias": (32,),
    "init_candidate_embed.2.weight": (EMB, 32), "init_candidate_embed.2.bias": (EMB,),
    "project_layer.0.weight": (256, 512), "project_layer.0.bias": (256,),
    "project_layer.2.weight": (EMB, 256), "project_layer.2.bias": (EMB,),
}
NOISY_IN_OUT = {"fc_h_v": (EMB, EMB), "fc_h_a": (EMB, EMB), "fc_z_v": (EMB, None), "fc_z_a": (EMB, None)}
NOISY_SUFFIXES = ("weight_mu", "weight_sigma", "weight_epsilon", "bias_mu", "bias_sigma", "bias_epsilon")
STATE_DICT_KEYS = tuple(PLAIN_SHAPES) + tuple("%s.%s" % (m, s) for m in NOISY for s in NOISY_SUFFIXES)

# irbpp_dqn_weights field -> state_dict key (NoisyLinear layers: the effective weight / bias)
_FIELDS = (("conv1_w", "heightEncoder.conv1.weight"), ("conv1_b", "heightEncoder.conv1.bias"),
           ("conv2_w", "heightEncoder.conv2.weight"), ("conv2_b", "heightEncoder.conv2.bias"),
           ("conv3_w", "heightEncoder.conv3.weight"), ("conv3_b", "heightEncoder.conv3.bias"),
           ("cand1_w", "init_candidate_embed.0.weight"), ("cand1_b", "init_candidate_embed.0.bias"),
           ("cand2_w", "init_candidate_embed.2.weight"), ("cand2_b", "init_candidate_embed.2.bias"),
           ("proj1_w", "project_layer.0.weight"), ("proj1_b", "project_layer.0.bias"),
           ("proj2_w", "project_layer.2.weight"), ("proj2_b", "project_layer.2.bias"),
           ("fc_h_v_w", "fc_h_v.weight"), ("fc_h_v_b", "fc_h_v.bias"), ("fc_z_v_w", "fc_z_v.weight"),
           ("fc_z_v_b", "fc_z_v.bias"), ("fc_h_a_w", "fc_h_a.weight"), ("fc_h_a_b", "fc_h_a.bias"),
           ("fc_z_a_w", "fc_z_a.weight"), ("fc_z_a_b", "fc_z_a.bias"))
SUPPORTED = "hidden_size 128, 1 <= atoms <= 32, selectedAction >= 1, a 32 x 32 heightmap (obs_len = sel * 5 + 9 + 1024)"


def check_state_dict(sd):
    """The number of atoms of a location-network state dict; ``ValueError`` for missing or misshapen keys."""
    missing = [k for k in STATE_DICT_KEYS if k not in sd]
    if missing:
        raise ValueError("state dict lacks %s (a location-level DQNBPP has the keys %s)" % (missing, list(STATE_DICT_KEYS)))
    zw = tuple(sd["fc_z_a.weight_mu"].shape)
    atoms = zw[0] if len(zw) == 2 else -1
    if not 1 <= atoms <= MAX_ATOMS:
        raise ValueError("fc_z_a has %d atoms; supported: %s" % (atoms, SUPPORTED))
    for k, shape in PLAIN_SHAPES.items():
        if tuple(sd[k].shape) != shape:
            raise ValueError("%s has shape %s, expected %s; supported: %s" % (k, tuple(sd[k].shape), shape, SUPPORTED))
    for m, (n_in, n_out) in NOISY_IN_OUT.items():
        n_out = atoms if n_out is None else n_out
        for s in NOISY_SUFFIXES:
            want = (n_out, n_in) if s.startswith("weight") else (n_out,)
            if tuple(sd["%s.%s" % (m, s)].shape) != want:
                raise ValueError("%s.%s has shape %s, expected %s; supported: %s" % (m, s, tuple(sd["%s.%s" % (m, s)].shape),
                                                                                   want, SUPPORTED))
    return atoms


class DeviceActor(object):
    """``Agent.act`` for every bin through ``irbpp_dqn_act``.

    ``net_or_state_dict``: a location-level ``DQNBPP`` (or any module with its ``state_dict`` keys, read live at every
    call) or a state dict (copied to the device once; ``train`` picks NoisyLinear's mode, default True as
    ``trainer.py`` acts).  ``clouds``: the ``DeviceShapeClouds`` that serves the next item's point-cloud feature (may be
    None when every call passes ``shape_feature=``).  ``support``: the atoms' values (``Agent.support``)."""

    def __init__(self, net_or_state_dict, clouds, support, train=None, device=None):
        import torch
        self._torch = torch
        self._lib = _lib.load()
        self.clouds = clouds
        if isinstance(net_or_state_dict, torch.nn.Module):
            self.net = net_or_state_dict
            if train is not None:
                raise ValueError("a module's mode is its training flag; train= is for state dicts")
            sd = self.net.state_dict()
        else:
            self.net = None
            sd = net_or_state_dict
            if not hasattr(sd, "keys"):
                raise ValueError("expected a DQNBPP module or its state dict, got %s" % type(sd).__name__)
            for k in STATE_DICT_KEYS:
                if k in sd and not isinstance(sd[k], torch.Tensor):
                    raise ValueError("state dict entry %s is not a tensor" % k)
        self.atoms = check_state_dict(sd)
        if not isinstance(support, torch.Tensor) or not support.is_cuda:
            raise ValueError("support must be a CUDA tensor of the %d atoms' values" % self.atoms)
        self.device = torch.device(device) if device is not None else support.device
        if support.device != self.device:
            raise ValueError("support lives on %s, the actor on %s" % (support.device, self.device))
        if support.numel() != self.atoms:
            raise ValueError("support has %d values, the network %d atoms" % (support.numel(), self.atoms))
        self.support = support.detach().to(torch.float32).reshape(-1).contiguous()
        if self.net is None:
            self.train = True if train is None else bool(train)
            self._static = {k: sd[k].detach().to(self.device, torch.float32).contiguous() for k in STATE_DICT_KEYS}
        self._scratch = None
        self._keep = None

    # ---- weights ----
    def _state(self):
        if self.net is None:
            return self._static, self.train
        sd = self.net.state_dict()
        for k in STATE_DICT_KEYS:
            if sd[k].device != self.device:
                raise ValueError("network weights live on %s, the actor on %s" % (sd[k].device, self.device))
        return sd, self.net.training

    def effective_weights(self):
        """The weights the kernels use, by field of ``irbpp_dqn_weights``: NoisyLinear layers with the torch expression
        of model.py:224-228 for the current mode (rebuilt at every call)."""
        torch = self._torch
        sd, train = self._state()
        out = {}
        with torch.no_grad():
            for m in NOISY:
                if train:
                    w = sd[m + ".weight_mu"] + sd[m + ".weight_sigma"] * sd[m + ".weight_epsilon"]
                    b = sd[m + ".bias_mu"] + sd[m + ".bias_sigma"] * sd[m + ".bias_epsilon"]
                else:
                    w, b = sd[m + ".weight_mu"], sd[m + ".bias_mu"]
                out[m + ".weight"], out[m + ".bias"] = w, b
            for k in PLAIN_SHAPES:
                out[k] = sd[k]
            ws = {f: out[k].detach().to(torch.float32).contiguous() for f, k in _FIELDS}
            enc = tuple(out[k].detach().to(torch.float32).contiguous() for k in (
                "shapeEncoder.linear1.weight", "shapeEncoder.linear1.bias", "shapeEncoder.linear2.weight",
                "shapeEncoder.linear2.bias"))
        return ws, enc

    # ---- the call ----
    def _check_state(self, state):
        torch = self._torch
        if not isinstance(state, torch.Tensor) or not state.is_cuda:
            raise ValueError("state must be a CUDA tensor [N, obs_len]")
        if state.device != self.device:
            raise ValueError("state lives on %s, the actor on %s" % (state.device, self.device))
        if state.dim() != 2 or state.dtype != torch.float32:
            raise ValueError("state must be float32 [N, obs_len], got %s %s" % (state.dtype, tuple(state.shape)))
        width = state.shape[1] - 9 - HM * HM
        if width < 5 or width % 5:
            raise ValueError("observation width %d is not selectedAction * 5 + 9 + 1024; supported: %s" % (state.shape[1], SUPPORTED))
        return state if state.stride(1) == 1 else state.contiguous(), width // 5

    def _run(self, state, mask, shape_feature, want_q):
        torch = self._torch
        state, sel = self._check_state(state)
        N = state.shape[0]
        ws, enc = self.effective_weights()
        if shape_feature is None:
            if self.clouds is None:
                raise ValueError("no DeviceShapeClouds given: pass shape_feature=")
            if self.clouds.item_col != sel * 5:
                raise ValueError("the point clouds read the item id at column %d, the observation carries it at %d"
                                 % (self.clouds.item_col, sel * 5))
            shape_feature = self.clouds.features(state, enc + (0.01,))
        if (not isinstance(shape_feature, torch.Tensor) or shape_feature.device != self.device
                or tuple(shape_feature.shape) != (N, EMB)):
            raise ValueError("shape_feature must be a tensor [%d, %d] on %s" % (N, EMB, self.device))
        shape_feature = shape_feature.detach().to(torch.float32).contiguous()
        m_ptr, m_row, m_elem = 0, 0, 0
        if mask is not None:
            if not isinstance(mask, torch.Tensor) or mask.device != self.device or tuple(mask.shape) != (N, sel):
                raise ValueError("mask must be a tensor [%d, %d] on %s" % (N, sel, self.device))
            if mask.dtype != torch.float32:
                mask = mask.to(torch.float32)
            m_ptr, m_row, m_elem = mask.data_ptr(), mask.stride(0), mask.stride(1)
        need = int(self._lib.irbpp_dqn_scratch_bytes(N, sel))
        if self._scratch is None or self._scratch.numel() < need:
            self._scratch = torch.empty(need, dtype=torch.uint8, device=self.device)
        actions = torch.empty(N, dtype=torch.int64, device=self.device)
        q = torch.empty((N, sel), dtype=torch.float32, device=self.device) if want_q else None
        w = _lib.IrbppDqnWeights(*([ws[f].data_ptr() for f, _ in _FIELDS] + [ctypes.c_float(0.01)]))
        rc = self._lib.irbpp_dqn_act(ctypes.byref(w), state.data_ptr(), state.stride(0), N, sel, shape_feature.data_ptr(),
                                     self.support.data_ptr(), self.atoms, m_ptr, m_row, m_elem, actions.data_ptr(),
                                     q.data_ptr() if q is not None else 0, self._scratch.data_ptr(), self._scratch.numel(),
                                     torch.cuda.current_stream(self.device).cuda_stream)
        _lib.check(self._lib, None, rc)
        self._keep = (ws, enc, shape_feature, mask, state)    # alive until the next call: the launches are asynchronous
        return actions, q

    def act(self, state, mask=None, shape_feature=None):
        """``Agent.act(state, mask)``: int64 ``[N]`` actions on the device.  ``mask=None`` masks nothing
        (agent.py:56)."""
        return self._run(state, mask, shape_feature, False)[0]

    def q_values(self, state, mask=None, shape_feature=None):
        """The masked ``sum_q_map`` of agent.py:53-57: float32 ``[N, sel]`` (-inf where ``mask != 1``)."""
        return self._run(state, mask, shape_feature, True)[1]
