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

``DeviceOrderActor`` does the same for the order network of the buffered configuration (``model.py:355-404``,
``args.level == 'order'``, ``csrc/irbpp_order_actor.cuh``), the first call of the hierarchical loop.
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


def _check_keys(sd, keys, plain_shapes, level, supported):
    """The number of atoms of a state dict; ``ValueError`` for missing or misshapen keys."""
    missing = [k for k in keys if k not in sd]
    if missing:
        raise ValueError("state dict lacks %s (a %s-level DQNBPP has the keys %s)" % (missing, level, list(keys)))
    zw = tuple(sd["fc_z_a.weight_mu"].shape)
    atoms = zw[0] if len(zw) == 2 else -1
    if not 1 <= atoms <= MAX_ATOMS:
        raise ValueError("fc_z_a has %d atoms; supported: %s" % (atoms, supported))
    for k, shape in plain_shapes.items():
        if tuple(sd[k].shape) != shape:
            raise ValueError("%s has shape %s, expected %s; supported: %s" % (k, tuple(sd[k].shape), shape, supported))
    for m, (n_in, n_out) in NOISY_IN_OUT.items():
        n_out = atoms if n_out is None else n_out
        for s in NOISY_SUFFIXES:
            want = (n_out, n_in) if s.startswith("weight") else (n_out,)
            if tuple(sd["%s.%s" % (m, s)].shape) != want:
                raise ValueError("%s.%s has shape %s, expected %s; supported: %s" % (m, s, tuple(sd["%s.%s" % (m, s)].shape),
                                                                                   want, supported))
    return atoms


def check_state_dict(sd):
    """The number of atoms of a location-network state dict; ``ValueError`` for missing or misshapen keys."""
    return _check_keys(sd, STATE_DICT_KEYS, PLAIN_SHAPES, "location", SUPPORTED)


# ---- the order level (model.py:355-383 with args.level == 'order', csrc/irbpp_order_actor.cuh) ----
MAX_BUFFER = 32
_ATT = "embedder.layers.0.0.module."
_FFN = "embedder.layers.0.1.module."
# key -> shape of the keys the order kernels read (init_candidate_embed and project_layer are in the reference's dict
# but unused at this level)
ORDER_PLAIN_SHAPES = dict(
    [(k, s) for k, s in PLAIN_SHAPES.items() if k.startswith(("heightEncoder.", "shapeEncoder."))] +
    [("gat_project_layer.0.weight", (256, 384)), ("gat_project_layer.0.bias", (256,)),
     ("gat_project_layer.2.weight", (EMB, 256)), ("gat_project_layer.2.bias", (EMB,)),
     (_ATT + "W_query.weight", (EMB, EMB)), (_ATT + "W_key.weight", (EMB, EMB)), (_ATT + "W_val.weight", (EMB, EMB)),
     (_ATT + "W_out.weight", (EMB, EMB)), (_ATT + "W_out.bias", (EMB,)),
     (_FFN + "0.weight", (EMB, EMB)), (_FFN + "0.bias", (EMB,)), (_FFN + "2.weight", (EMB, EMB)), (_FFN + "2.bias", (EMB,))])
ORDER_STATE_DICT_KEYS = tuple(ORDER_PLAIN_SHAPES) + tuple("%s.%s" % (m, s) for m in NOISY for s in NOISY_SUFFIXES)
# irbpp_dqn_order_weights field -> state_dict key
_ORDER_FIELDS = (_FIELDS[:6] + (
    ("gat1_w", "gat_project_layer.0.weight"), ("gat1_b", "gat_project_layer.0.bias"),
    ("gat2_w", "gat_project_layer.2.weight"), ("gat2_b", "gat_project_layer.2.bias"),
    ("wq", _ATT + "W_query.weight"), ("wk", _ATT + "W_key.weight"), ("wv", _ATT + "W_val.weight"),
    ("wo_w", _ATT + "W_out.weight"), ("wo_b", _ATT + "W_out.bias"), ("ff1_w", _FFN + "0.weight"), ("ff1_b", _FFN + "0.bias"),
    ("ff2_w", _FFN + "2.weight"), ("ff2_b", _FFN + "2.bias")) + _FIELDS[14:])
ORDER_SUPPORTED = ("hidden_size 128, one attention head and layer with feed-forward width 128, 2 <= bufferSize <= 32, "
                   "1 <= atoms <= 32, a 32 x 32 heightmap (obs_len = bufferSize + 1024)")


def check_order_state_dict(sd):
    """The number of atoms of an order-network state dict; ``ValueError`` for missing or misshapen keys."""
    return _check_keys(sd, ORDER_STATE_DICT_KEYS, ORDER_PLAIN_SHAPES, "order", ORDER_SUPPORTED)


class _NetworkSource(object):
    """The weights a device actor reads: a module (read live at every call, its ``training`` flag picks NoisyLinear's
    mode) or a state dict (copied to the device once, ``train`` picks the mode, default True).  ``keys``: the state
    dict keys the kernels read; ``check(sd)`` validates them and returns the number of atoms."""

    def __init__(self, net_or_state_dict, support, train, device, keys, check):
        import torch
        self._torch = torch
        self._lib = _lib.load()
        self._keys = keys
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
            for k in keys:
                if k in sd and not isinstance(sd[k], torch.Tensor):
                    raise ValueError("state dict entry %s is not a tensor" % k)
        self.atoms = check(sd)
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
            self._static = {k: sd[k].detach().to(self.device, torch.float32).contiguous() for k in keys}
        self._scratch = None
        self._keep = None

    def _state(self):
        if self.net is None:
            return self._static, self.train
        sd = self.net.state_dict()
        for k in self._keys:
            if sd[k].device != self.device:
                raise ValueError("network weights live on %s, the actor on %s" % (sd[k].device, self.device))
        return sd, self.net.training

    def _effective(self, plain):
        """The state dict's ``plain`` keys and, for every NoisyLinear layer m, ``m.weight`` / ``m.bias`` built with the
        torch expression of model.py:224-228 for the current mode (at every call)."""
        sd, train = self._state()
        out = {}
        with self._torch.no_grad():
            for m in NOISY:
                if train:
                    w = sd[m + ".weight_mu"] + sd[m + ".weight_sigma"] * sd[m + ".weight_epsilon"]
                    b = sd[m + ".bias_mu"] + sd[m + ".bias_sigma"] * sd[m + ".bias_epsilon"]
                else:
                    w, b = sd[m + ".weight_mu"], sd[m + ".bias_mu"]
                out[m + ".weight"], out[m + ".bias"] = w, b
            for k in plain:
                out[k] = sd[k]
        return out

    def _target_inputs(self, N, next_actions, returns, nonterminals, v_min, v_max, with_p):
        """The target pass's per-transition inputs as contiguous device vectors, and its outputs ``m`` and ``p_next``
        (None unless ``with_p``)."""
        torch = self._torch
        if self.atoms < 2:
            raise ValueError("the target distribution needs 2 <= atoms <= %d (the network has %d)" % (MAX_ATOMS, self.atoms))
        if not float(v_max) > float(v_min):
            raise ValueError("need v_max > v_min, got v_min %r, v_max %r" % (v_min, v_max))
        out = []
        for name, x, dtype in (("next_actions", next_actions, torch.int64), ("returns", returns, torch.float32),
                               ("nonterminals", nonterminals, torch.float32)):
            if not isinstance(x, torch.Tensor) or x.device != self.device or x.numel() != N:
                raise ValueError("%s must be a tensor of %d values on %s" % (name, N, self.device))
            out.append(x.detach().reshape(N).to(dtype).contiguous())
        m = torch.empty((N, self.atoms), dtype=torch.float32, device=self.device)
        p = torch.empty((N, self.atoms), dtype=torch.float32, device=self.device) if with_p else None
        return out + [m, p]

    def _scratch_of(self, need):
        if self._scratch is None or self._scratch.numel() < need:
            self._scratch = self._torch.empty(need, dtype=self._torch.uint8, device=self.device)
        return self._scratch


class DeviceActor(_NetworkSource):
    """``Agent.act`` for every bin through ``irbpp_dqn_act``.

    ``net_or_state_dict``: a location-level ``DQNBPP`` (or any module with its ``state_dict`` keys, read live at every
    call) or a state dict (copied to the device once; ``train`` picks NoisyLinear's mode, default True as
    ``trainer.py`` acts).  ``clouds``: the ``DeviceShapeClouds`` that serves the next item's point-cloud feature (may be
    None when every call passes ``shape_feature=``).  ``support``: the atoms' values (``Agent.support``)."""

    def __init__(self, net_or_state_dict, clouds, support, train=None, device=None):
        _NetworkSource.__init__(self, net_or_state_dict, support, train, device, STATE_DICT_KEYS, check_state_dict)
        self.clouds = clouds

    # ---- weights ----
    def effective_weights(self):
        """The weights the kernels use, by field of ``irbpp_dqn_weights``: NoisyLinear layers with the torch expression
        of model.py:224-228 for the current mode (rebuilt at every call)."""
        torch = self._torch
        with torch.no_grad():
            out = self._effective(PLAIN_SHAPES)
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

    def _inputs(self, state, shape_feature):
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
        w = _lib.IrbppDqnWeights(*([ws[f].data_ptr() for f, _ in _FIELDS] + [ctypes.c_float(0.01)]))
        return state, sel, N, ws, enc, shape_feature, w

    def _run(self, state, mask, shape_feature, want_q):
        torch = self._torch
        state, sel, N, ws, enc, shape_feature, w = self._inputs(state, shape_feature)
        m_ptr, m_row, m_elem = 0, 0, 0
        if mask is not None:
            if not isinstance(mask, torch.Tensor) or mask.device != self.device or tuple(mask.shape) != (N, sel):
                raise ValueError("mask must be a tensor [%d, %d] on %s" % (N, sel, self.device))
            if mask.dtype != torch.float32:
                mask = mask.to(torch.float32)
            m_ptr, m_row, m_elem = mask.data_ptr(), mask.stride(0), mask.stride(1)
        self._scratch_of(int(self._lib.irbpp_dqn_scratch_bytes(N, sel)))
        actions = torch.empty(N, dtype=torch.int64, device=self.device)
        q = torch.empty((N, sel), dtype=torch.float32, device=self.device) if want_q else None
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

    def target(self, next_state, next_actions, returns, nonterminals, v_min, v_max, discount_n, shape_feature=None,
               with_p=True):
        """The target distribution of ``Agent.learn`` (agent.py:94-115) through ``irbpp_dqn_target``, with this actor's
        network as the target net: ``p_next = p(s', a*)`` and ``m``, the projection of ``returns + nonterminals *
        discount_n * z`` onto the support, both float32 ``[B, atoms]`` on the device.  ``next_actions``: a* of the
        online net (``online_actor.act(next_state)``, unmasked as agent.py:90-92), clamped to the rows;
        ``returns`` ``[B]`` and ``nonterminals`` ``[B, 1]`` as ``PrioritizedReplayBank.sample`` returns them.
        ``with_p=False`` skips ``p_next`` (returned as None)."""
        torch = self._torch
        state, sel, B, ws, enc, shape_feature, w = self._inputs(next_state, shape_feature)
        a, r, nt, m, p = self._target_inputs(B, next_actions, returns, nonterminals, v_min, v_max, with_p)
        p_ptr = p.data_ptr() if p is not None else None
        self._scratch_of(int(self._lib.irbpp_dqn_scratch_bytes(B, sel)))
        rc = self._lib.irbpp_dqn_target(ctypes.byref(w), state.data_ptr(), state.stride(0), B, sel, shape_feature.data_ptr(),
                                        self.support.data_ptr(), self.atoms, a.data_ptr(), r.data_ptr(), nt.data_ptr(),
                                        float(discount_n), float(v_min), float(v_max), m.data_ptr(), p_ptr,
                                        self._scratch.data_ptr(), self._scratch.numel(),
                                        torch.cuda.current_stream(self.device).cuda_stream)
        _lib.check(self._lib, None, rc)
        self._keep = (ws, enc, shape_feature, state, a, r, nt)
        return m, p

    def log_prob(self, states, actions):
        """``online_net(states, log=True)[arange(B), actions]`` of ``Agent.learn``'s gradient pass (agent.py:85-86):
        float32 ``[B, atoms]``, differentiable with respect to every parameter of the live module the forward pass uses.
        torch computes the height encoder, the shape encoder on ``clouds.sample(states)`` and the NoisyLinear effective
        weights with autograd; ``irbpp_dqn_log_prob`` / ``irbpp_dqn_log_prob_backward`` run the candidate-row network
        and its backward pass.  ``actions`` (a_t, ``[B]``) are clamped to the rows, where the reference raises
        ``IndexError``.  Double backward is not supported."""
        torch = self._torch
        if self.net is None:
            raise ValueError("log_prob trains the live module; a state-dict actor has no parameters")
        state, sel = self._check_state(states)
        B = state.shape[0]
        if not isinstance(actions, torch.Tensor) or actions.device != self.device or actions.numel() != B:
            raise ValueError("actions must be a tensor of %d values on %s" % (B, self.device))
        if self.clouds is None:
            raise ValueError("log_prob samples the next item's points: the actor needs a DeviceShapeClouds")
        if self.clouds.item_col != sel * 5:
            raise ValueError("the point clouds read the item id at column %d, the observation carries it at %d"
                             % (self.clouds.item_col, sel * 5))
        self._state()                                            # the weights' device
        net = self.net
        params = dict(net.named_parameters())
        params.update(net.named_buffers())
        eff = {}
        for m in NOISY:                                          # model.py:224-228, with autograd
            if net.training:
                eff[m + ".weight"] = params[m + ".weight_mu"] + params[m + ".weight_sigma"] * params[m + ".weight_epsilon"]
                eff[m + ".bias"] = params[m + ".bias_mu"] + params[m + ".bias_sigma"] * params[m + ".bias_epsilon"]
            else:
                eff[m + ".weight"], eff[m + ".bias"] = params[m + ".weight_mu"], params[m + ".bias_mu"]
        weights = [(eff[k] if k in eff else params[k]).to(torch.float32).contiguous() for _, k in _ROW_FIELDS]
        hm = state[:, sel * 5 + 9:sel * 5 + 9 + HM * HM].reshape(B, 1, HM, HM)
        map_feature = net.heightEncoder(hm).reshape(B, -1)                            # model.py:326-327
        shape_feature = net.shapeEncoder(self.clouds.sample(state)).max(1)[0]          # model.py:329-335
        a = actions.detach().reshape(B).to(torch.int64).contiguous()
        return _log_prob_function().apply(self, state, sel, a, shape_feature.to(torch.float32).contiguous(),
                                          map_feature.to(torch.float32).contiguous(), *weights)


# the row-section fields of irbpp_dqn_weights: the tensors irbpp_dqn_log_prob reads and irbpp_dqn_grads returns
_ROW_FIELDS = _FIELDS[6:]
_LOG_PROB = []


def _log_prob_function():
    """The ``torch.autograd.Function`` behind ``DeviceActor.log_prob`` (built once; torch is imported lazily here)."""
    if _LOG_PROB:
        return _LOG_PROB[0]
    import torch

    def weights_struct(ws):
        ptrs = dict((f, t.data_ptr()) for (f, _), t in zip(_ROW_FIELDS, ws))
        return _lib.IrbppDqnWeights(*([ptrs.get(f, 0) for f, _ in _FIELDS] + [ctypes.c_float(0.01)]))

    class LogProb(torch.autograd.Function):
        @staticmethod
        def forward(ctx, actor, state, sel, actions, shape_feature, map_feature, *ws):
            B = state.shape[0]
            lib = actor._lib
            w = weights_struct(ws)
            scratch = actor._scratch_of(int(lib.irbpp_dqn_log_prob_scratch_bytes(B, sel)))
            log_p = torch.empty((B, actor.atoms), dtype=torch.float32, device=actor.device)
            rc = lib.irbpp_dqn_log_prob(ctypes.byref(w), state.data_ptr(), state.stride(0), B, sel,
                                        shape_feature.data_ptr(), map_feature.data_ptr(), actions.data_ptr(), actor.atoms,
                                        log_p.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                        torch.cuda.current_stream(actor.device).cuda_stream)
            _lib.check(lib, None, rc)
            ctx.actor, ctx.state, ctx.sel, ctx.actions = actor, state, sel, actions
            ctx.save_for_backward(shape_feature, map_feature, *ws)
            return log_p

        @staticmethod
        @torch.autograd.function.once_differentiable
        def backward(ctx, grad):
            actor, state, sel, actions = ctx.actor, ctx.state, ctx.sel, ctx.actions
            shape_feature, map_feature = ctx.saved_tensors[:2]
            ws = ctx.saved_tensors[2:]
            B, lib = state.shape[0], actor._lib
            grad = grad.to(torch.float32).contiguous()
            w = weights_struct(ws)
            dws = [torch.empty_like(t) for t in ws]
            g = _lib.IrbppDqnGrads(*[t.data_ptr() for t in dws])
            d_sf, d_mf = torch.empty_like(shape_feature), torch.empty_like(map_feature)
            scratch = actor._scratch_of(int(lib.irbpp_dqn_log_prob_scratch_bytes(B, sel)))
            rc = lib.irbpp_dqn_log_prob_backward(ctypes.byref(w), state.data_ptr(), state.stride(0), B, sel,
                                                 shape_feature.data_ptr(), map_feature.data_ptr(), actions.data_ptr(),
                                                 actor.atoms, grad.data_ptr(), ctypes.byref(g), d_sf.data_ptr(),
                                                 d_mf.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                                 torch.cuda.current_stream(actor.device).cuda_stream)
            _lib.check(lib, None, rc)
            actor._keep = (grad, ws, state, actions)             # alive until the next call: the launches are asynchronous
            return (None, None, None, None, d_sf, d_mf) + tuple(dws)

    _LOG_PROB.append(LogProb)
    return LogProb


class DeviceOrderActor(_NetworkSource):
    """``Agent.act`` of the order network (``DQNBPP`` with ``args.level == 'order'``, ``bufferSize`` k > 1) for every
    bin through ``irbpp_dqn_order_act``: the first call of the hierarchical loop (``trainer.py:261-281``,
    ``tools.py:361-387``)::

        order_actor = DeviceOrderActor(orderDQN.online_net, clouds, orderDQN.support)
        orderAction = order_actor.act(orderState)        # drop-in for orderDQN.act(orderState, None)

    ``net_or_state_dict``, ``train`` and ``support`` as for ``DeviceActor``.  ``clouds``: the ``DeviceShapeClouds`` (or
    ``pointnet.OrderShapeClouds``, the order level's own point rule) whose ``features`` on the ids ``arange(S)`` give the
    per-shape table the kernels gather from, one index set per act; may be None when every call passes
    ``shape_features=`` (float32 ``[S, 128]`` on the actor's device)."""

    def __init__(self, net_or_state_dict, clouds, support, train=None, device=None):
        _NetworkSource.__init__(self, net_or_state_dict, support, train, device, ORDER_STATE_DICT_KEYS,
                                check_order_state_dict)
        self.clouds = clouds

    def effective_weights(self):
        """The weights the kernels use, by field of ``irbpp_dqn_order_weights``, and the shape encoder's tensors."""
        torch = self._torch
        with torch.no_grad():
            out = self._effective(ORDER_PLAIN_SHAPES)
            ws = {f: out[k].detach().to(torch.float32).contiguous() for f, k in _ORDER_FIELDS}
            enc = tuple(out[k].detach().to(torch.float32).contiguous() for k in (
                "shapeEncoder.linear1.weight", "shapeEncoder.linear1.bias", "shapeEncoder.linear2.weight",
                "shapeEncoder.linear2.bias"))
        return ws, enc

    def _check_state(self, state):
        torch = self._torch
        if not isinstance(state, torch.Tensor) or not state.is_cuda:
            raise ValueError("order state must be a CUDA tensor [N, bufferSize + 1024]")
        if state.device != self.device:
            raise ValueError("order state lives on %s, the actor on %s" % (state.device, self.device))
        if state.dim() != 2 or state.dtype != torch.float32:
            raise ValueError("order state must be float32 [N, bufferSize + 1024], got %s %s" % (state.dtype, tuple(state.shape)))
        k = state.shape[1] - HM * HM
        if not 2 <= k <= MAX_BUFFER:
            raise ValueError("order observation width %d is not bufferSize + 1024; supported: %s" % (state.shape[1], ORDER_SUPPORTED))
        return state if state.stride(1) == 1 else state.contiguous(), k

    def _inputs(self, state, shape_features):
        torch = self._torch
        state, k = self._check_state(state)
        N = state.shape[0]
        ws, enc = self.effective_weights()
        if shape_features is None:
            if self.clouds is None:
                raise ValueError("no DeviceShapeClouds given: pass shape_features=")
            ids = torch.arange(self.clouds.S, dtype=torch.int32, device=self.device)
            shape_features = self.clouds.features(ids, enc + (0.01,))
        if (not isinstance(shape_features, torch.Tensor) or shape_features.device != self.device
                or shape_features.dim() != 2 or shape_features.shape[1] != EMB or shape_features.shape[0] < 1):
            raise ValueError("shape_features must be a tensor [S, %d] on %s" % (EMB, self.device))
        shape_features = shape_features.detach().to(torch.float32).contiguous()
        w = _lib.IrbppDqnOrderWeights(*([ws[f].data_ptr() for f, _ in _ORDER_FIELDS] + [ctypes.c_float(0.01)]))
        return state, k, N, ws, enc, shape_features, w

    def _run(self, state, mask, shape_features, want_q):
        torch = self._torch
        state, k, N, ws, enc, shape_features, w = self._inputs(state, shape_features)
        S = shape_features.shape[0]
        m_ptr, m_row, m_elem = 0, 0, 0
        if mask is not None:
            if not isinstance(mask, torch.Tensor) or mask.device != self.device or tuple(mask.shape) != (N, k):
                raise ValueError("mask must be a tensor [%d, %d] on %s" % (N, k, self.device))
            if mask.dtype != torch.float32:
                mask = mask.to(torch.float32)
            m_ptr, m_row, m_elem = mask.data_ptr(), mask.stride(0), mask.stride(1)
        scratch = self._scratch_of(int(self._lib.irbpp_dqn_order_scratch_bytes(N, k, S)))
        actions = torch.empty(N, dtype=torch.int64, device=self.device)
        q = torch.empty((N, k), dtype=torch.float32, device=self.device) if want_q else None
        rc = self._lib.irbpp_dqn_order_act(ctypes.byref(w), state.data_ptr(), state.stride(0), N, k, shape_features.data_ptr(),
                                           S, self.support.data_ptr(), self.atoms, m_ptr, m_row, m_elem, actions.data_ptr(),
                                           q.data_ptr() if q is not None else 0, scratch.data_ptr(), scratch.numel(),
                                           torch.cuda.current_stream(self.device).cuda_stream)
        _lib.check(self._lib, None, rc)
        self._keep = (ws, enc, shape_features, mask, state)    # alive until the next call: the launches are asynchronous
        return actions, q

    def act(self, order_state, mask=None, shape_features=None):
        """``orderDQN.act(orderState, mask)``: int64 ``[N]`` slots on the device.  ``mask=None`` masks nothing, as the
        reference acts at this level."""
        return self._run(order_state, mask, shape_features, False)[0]

    def q_values(self, order_state, mask=None, shape_features=None):
        """The masked ``sum_q_map`` of agent.py:53-57: float32 ``[N, k]`` (-inf where ``mask != 1``)."""
        return self._run(order_state, mask, shape_features, True)[1]

    def target(self, next_state, next_actions, returns, nonterminals, v_min, v_max, discount_n, shape_features=None,
               with_p=True):
        """``DeviceActor.target`` at the order level, through ``irbpp_dqn_order_target``: ``(m, p_next)`` for the
        order network's ``learn`` (trainer.py:318), a* clamped to the k slots."""
        torch = self._torch
        state, k, B, ws, enc, shape_features, w = self._inputs(next_state, shape_features)
        S = shape_features.shape[0]
        a, r, nt, m, p = self._target_inputs(B, next_actions, returns, nonterminals, v_min, v_max, with_p)
        p_ptr = p.data_ptr() if p is not None else None
        scratch = self._scratch_of(int(self._lib.irbpp_dqn_order_scratch_bytes(B, k, S)))
        rc = self._lib.irbpp_dqn_order_target(ctypes.byref(w), state.data_ptr(), state.stride(0), B, k,
                                              shape_features.data_ptr(), S, self.support.data_ptr(), self.atoms,
                                              a.data_ptr(), r.data_ptr(), nt.data_ptr(), float(discount_n), float(v_min),
                                              float(v_max), m.data_ptr(), p_ptr, scratch.data_ptr(),
                                              scratch.numel(), torch.cuda.current_stream(self.device).cuda_stream)
        _lib.check(self._lib, None, rc)
        self._keep = (ws, enc, shape_features, state, a, r, nt)
        return m, p

    def log_prob(self, states, actions):
        """``online_net(states, log=True)[arange(B), actions]`` of the order network's ``learn`` (agent.py:85-86,
        trainer.py:318): float32 ``[B, atoms]``, differentiable with respect to every parameter of the live module the
        forward pass uses.  torch computes the height encoder, the shape encoder on ``clouds.sample(arange(S))`` (one
        index set for the batch, as act draws it) and the NoisyLinear effective weights with autograd;
        ``irbpp_dqn_order_log_prob`` / ``irbpp_dqn_order_log_prob_backward`` run everything per slot and per bin and its
        backward pass.  ``actions`` (a_t, ``[B]``) are clamped to the k slots and item ids to the library, where the
        reference raises ``IndexError``.  Double backward is not supported."""
        torch = self._torch
        if self.net is None:
            raise ValueError("log_prob trains the live module; a state-dict actor has no parameters")
        state, k = self._check_state(states)
        B = state.shape[0]
        if not isinstance(actions, torch.Tensor) or actions.device != self.device or actions.numel() != B:
            raise ValueError("actions must be a tensor of %d values on %s" % (B, self.device))
        if self.clouds is None:
            raise ValueError("log_prob samples every library shape's points: the actor needs a DeviceShapeClouds")
        self._state()                                            # the weights' device
        net = self.net
        params = dict(net.named_parameters())
        params.update(net.named_buffers())
        eff = {}
        for m in NOISY:                                          # model.py:224-228, with autograd
            if net.training:
                eff[m + ".weight"] = params[m + ".weight_mu"] + params[m + ".weight_sigma"] * params[m + ".weight_epsilon"]
                eff[m + ".bias"] = params[m + ".bias_mu"] + params[m + ".bias_sigma"] * params[m + ".bias_epsilon"]
            else:
                eff[m + ".weight"], eff[m + ".bias"] = params[m + ".weight_mu"], params[m + ".bias_mu"]
        weights = [(eff[key] if key in eff else params[key]).to(torch.float32).contiguous() for _, key in _ORDER_ROW_FIELDS]
        hm = state[:, k:k + HM * HM].reshape(B, 1, HM, HM)
        map_feature = net.heightEncoder(hm).reshape(B, -1)                            # model.py:361-363
        ids = torch.arange(self.clouds.S, dtype=torch.int32, device=self.device)
        shape_features = net.shapeEncoder(self.clouds.sample(ids)).max(1)[0]         # model.py:365-372, per shape
        a = actions.detach().reshape(B).to(torch.int64).contiguous()
        return _order_log_prob_function().apply(self, state, k, a, shape_features.to(torch.float32).contiguous(),
                                                map_feature.to(torch.float32).contiguous(), *weights)


# the fields of irbpp_dqn_order_weights after the convolutions: the tensors irbpp_dqn_order_log_prob reads and
# irbpp_dqn_order_grads returns
_ORDER_ROW_FIELDS = _ORDER_FIELDS[6:]
_ORDER_LOG_PROB = []


def _order_log_prob_function():
    """The ``torch.autograd.Function`` behind ``DeviceOrderActor.log_prob`` (built once; torch is imported lazily)."""
    if _ORDER_LOG_PROB:
        return _ORDER_LOG_PROB[0]
    import torch

    def weights_struct(ws):
        ptrs = dict((f, t.data_ptr()) for (f, _), t in zip(_ORDER_ROW_FIELDS, ws))
        return _lib.IrbppDqnOrderWeights(*([ptrs.get(f, 0) for f, _ in _ORDER_FIELDS] + [ctypes.c_float(0.01)]))

    class OrderLogProb(torch.autograd.Function):
        @staticmethod
        def forward(ctx, actor, state, k, actions, shape_features, map_feature, *ws):
            B, S = state.shape[0], shape_features.shape[0]
            lib = actor._lib
            w = weights_struct(ws)
            scratch = actor._scratch_of(int(lib.irbpp_dqn_order_log_prob_scratch_bytes(B, k, S)))
            log_p = torch.empty((B, actor.atoms), dtype=torch.float32, device=actor.device)
            rc = lib.irbpp_dqn_order_log_prob(ctypes.byref(w), state.data_ptr(), state.stride(0), B, k,
                                              shape_features.data_ptr(), S, map_feature.data_ptr(), actions.data_ptr(),
                                              actor.atoms, log_p.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                              torch.cuda.current_stream(actor.device).cuda_stream)
            _lib.check(lib, None, rc)
            ctx.actor, ctx.state, ctx.k, ctx.actions = actor, state, k, actions
            ctx.save_for_backward(shape_features, map_feature, *ws)
            return log_p

        @staticmethod
        @torch.autograd.function.once_differentiable
        def backward(ctx, grad):
            actor, state, k, actions = ctx.actor, ctx.state, ctx.k, ctx.actions
            shape_features, map_feature = ctx.saved_tensors[:2]
            ws = ctx.saved_tensors[2:]
            B, S, lib = state.shape[0], shape_features.shape[0], actor._lib
            grad = grad.to(torch.float32).contiguous()
            w = weights_struct(ws)
            dws = [torch.empty_like(t) for t in ws]
            g = _lib.IrbppDqnOrderGrads(*[t.data_ptr() for t in dws])
            d_sf, d_mf = torch.empty_like(shape_features), torch.empty_like(map_feature)
            scratch = actor._scratch_of(int(lib.irbpp_dqn_order_log_prob_scratch_bytes(B, k, S)))
            rc = lib.irbpp_dqn_order_log_prob_backward(ctypes.byref(w), state.data_ptr(), state.stride(0), B, k,
                                                       shape_features.data_ptr(), S, map_feature.data_ptr(),
                                                       actions.data_ptr(), actor.atoms, grad.data_ptr(), ctypes.byref(g),
                                                       d_sf.data_ptr(), d_mf.data_ptr(), scratch.data_ptr(),
                                                       scratch.numel(), torch.cuda.current_stream(actor.device).cuda_stream)
            _lib.check(lib, None, rc)
            actor._keep = (grad, ws, state, actions)             # alive until the next call: the launches are asynchronous
            return (None, None, None, None, d_sf, d_mf) + tuple(dws)

    _ORDER_LOG_PROB.append(OrderLogProb)
    return OrderLogProb
