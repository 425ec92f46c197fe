"""``Agent.learn`` (reference ``agent.py:68-125``) restated on ``DQNPort`` / ``OrderDQNPort`` -- TEST INFRASTRUCTURE:
the checker of ``irbpp_dqn_target`` / ``irbpp_dqn_order_target`` and of ``learner_glue.device_learn``.

* ``distribution``   the network's atom distribution (``model.py:393-400``), ``log=True`` for the log-softmax of
  ``agent.py:85``;
* ``project64``      ``agent.py:100-115`` in float64 NumPy: ``Tz``, ``b``, ``l`` / ``u`` with both fix-ups, ``m``;
* ``target64``       the double-Q target in float64: a* from the online net (or an override, so that a kernel's a* on a
  near-tie can be fed in), ``p(s', a*)`` from the target net, the projection and, given ``log_ps_a``, the loss;
* ``torch_projection`` and ``learn_step32``  the reference's float32 torch expressions of ``agent.py:84-121`` on the
  port modules (``index_add_`` and all), the step ``device_learn`` is compared with;
* ``ReferenceDQN`` / ``ReferenceOrderDQN``  ports with the reference's ``forward(x, log=False)`` (``model.py:386-404``):
  the shape features are computed with gradients from ``DeviceShapeClouds.sample`` and the module's own
  ``shapeEncoder``, so ``device_learn`` can call them exactly as it calls the reference's ``DQNBPP``.
"""
import copy

import numpy as np
import torch
from torch.nn import functional as F
from torch.nn.utils import clip_grad_norm_

from oracle.dqn_port import DQNPort
from oracle.order_dqn_port import OrderDQNPort


def distribution(net, obs, shape_feature, log=False):
    """``q = v + a - mean a`` through softmax (or log_softmax) over the atoms: ``[B, rows, atoms]``."""
    e, g = net.embed(obs, shape_feature)
    v = net.fc_z_v(F.relu(net.fc_h_v(g)))[:, None, :]
    a = net.advantage(e)
    q = v + a - a.mean(1, keepdim=True)
    return F.log_softmax(q, dim=2) if log else F.softmax(q, dim=2)


def project64(p, returns, nonterminals, support, v_min, v_max, discount_n):
    """agent.py:100-115 in float64: dict of ``Tz``, ``b``, ``l``, ``u`` (after the fix-ups) and ``m``, all ``[B, atoms]``."""
    p = np.asarray(p, np.float64)
    B, atoms = p.shape
    z = np.asarray(support, np.float64).reshape(1, atoms)
    R = np.asarray(returns, np.float64).reshape(B, 1)
    nt = np.asarray(nonterminals, np.float64).reshape(B, 1)
    Tz = np.clip(R + nt * float(discount_n) * z, v_min, v_max)
    b = (Tz - v_min) / ((v_max - v_min) / (atoms - 1))
    l, u = np.floor(b).astype(np.int64), np.ceil(b).astype(np.int64)
    l[(u > 0) & (l == u)] -= 1
    u[(l < atoms - 1) & (l == u)] += 1
    m = np.zeros((B, atoms))
    rows = np.broadcast_to(np.arange(B)[:, None], (B, atoms))
    np.add.at(m, (rows, l), p * (u - b))
    np.add.at(m, (rows, u), p * (b - l))
    return dict(Tz=Tz, b=b, l=l, u=u, m=m)


def target64(online, target, next_obs, sf_online, sf_target, support, returns, nonterminals, v_min, v_max, discount_n,
             next_actions=None, log_ps_a=None):
    """agent.py:88-117 in float64 on copies of the two port modules (their modes and noise kept).  ``next_actions``
    overrides the online argmax.  Returns dict of ``a_star``, ``p`` and ``project64``'s entries, and ``loss`` when
    ``log_ps_a`` is given."""
    t = lambda x: torch.as_tensor(np.asarray(x) if not isinstance(x, torch.Tensor) else x).double()
    with torch.no_grad():
        obs = t(next_obs)
        dev = obs.device
        tg = copy.deepcopy(target).to(dev, torch.float64)
        z = t(support).to(dev)
        if next_actions is None:
            on = copy.deepcopy(online).to(dev, torch.float64)
            a_star = (distribution(on, obs, t(sf_online).to(dev)) * z).sum(2).argmax(1)
        else:
            a_star = torch.as_tensor(next_actions, device=dev).long()
        p = distribution(tg, obs, t(sf_target).to(dev))[torch.arange(obs.shape[0], device=dev), a_star]
    out = project64(p.cpu().numpy(), t(returns).cpu().numpy(), t(nonterminals).cpu().numpy(), z.cpu().numpy(),
                    v_min, v_max, discount_n)
    out.update(a_star=a_star.cpu().numpy(), p=p.cpu().numpy())
    if log_ps_a is not None:
        out["loss"] = -(out["m"] * np.asarray(log_ps_a, np.float64)).sum(1)
    return out


def torch_projection(pns_a, returns, nonterminals, support, v_min, v_max, discount_n):
    """agent.py:100-115 as the reference writes it, on the tensors' device and dtype."""
    B, atoms = pns_a.shape
    delta_z = (v_max - v_min) / (atoms - 1)
    Tz = returns.reshape(B).unsqueeze(1) + nonterminals.reshape(B, 1) * discount_n * support.unsqueeze(0)
    Tz = Tz.clamp(min=v_min, max=v_max)
    b = (Tz - v_min) / delta_z
    l, u = b.floor().to(torch.int64), b.ceil().to(torch.int64)
    l[(u > 0) * (l == u)] -= 1
    u[(l < (atoms - 1)) * (l == u)] += 1
    m = pns_a.new_zeros(B, atoms)
    offset = torch.linspace(0, ((B - 1) * atoms), B, device=pns_a.device).unsqueeze(1).expand(B, atoms).to(torch.int64)
    m.view(-1).index_add_(0, (l + offset).view(-1), (pns_a * (u.float() - b)).view(-1))
    m.view(-1).index_add_(0, (u + offset).view(-1), (pns_a * (b - l.float())).view(-1))
    return m


def learn_step32(online, target, optimiser, norm_clip, batch, sf_states, sf_next_target, support, v_min, v_max,
                 discount_n, next_actions):
    """agent.py:84-121 in float32 torch on the port modules with the given a*: ``batch`` is ``(states, actions,
    returns, next_states, nonterminals, weights)``; ``sf_states`` carries the gradient pass's shape features (with
    gradients when the shape encoder is to be trained).  Returns ``(loss, m)``; steps ``optimiser``."""
    states, actions, returns, next_states, nonterminals, weights = batch
    B = states.shape[0]
    log_ps = distribution(online, states, sf_states, log=True)
    log_ps_a = log_ps[torch.arange(B, device=states.device), actions]
    with torch.no_grad():
        pns_a = distribution(target, next_states, sf_next_target)[torch.arange(B, device=states.device), next_actions]
        m = torch_projection(pns_a, returns, nonterminals, support, v_min, v_max, discount_n)
    loss = -torch.sum(m * log_ps_a, 1)
    online.zero_grad()
    (weights * loss).mean().backward()
    clip_grad_norm_(online.parameters(), norm_clip)
    optimiser.step()
    return loss.detach(), m


class _Shared(object):
    """Holds an object that every copy of the module shares (``copy.deepcopy`` returns the holder itself)."""

    def __init__(self, obj):
        self.obj = obj

    def __deepcopy__(self, memo):
        return self


class _ReferenceForward(object):
    """``forward(x, log=False)`` of model.py:386-404 over ``self.clouds`` (one point index set per call)."""

    @property
    def clouds(self):
        return self._clouds.obj

    def shape_features_of(self, x):
        if isinstance(self, OrderDQNPort):          # every library shape, one index set (model.py:365-372)
            ids = torch.arange(self.clouds.S, dtype=torch.int32, device=x.device)
            return self.shape_feature(self.clouds.sample(ids))
        return self.shape_feature(self.clouds.sample(x))

    def forward(self, x, log=False):
        return distribution(self, x, self.shape_features_of(x), log)


class ReferenceDQN(_ReferenceForward, DQNPort):
    def __init__(self, clouds, **kw):
        DQNPort.__init__(self, **kw)
        self._clouds = _Shared(clouds)


class ReferenceOrderDQN(_ReferenceForward, OrderDQNPort):
    def __init__(self, clouds, **kw):
        OrderDQNPort.__init__(self, **kw)
        self._clouds = _Shared(clouds)
