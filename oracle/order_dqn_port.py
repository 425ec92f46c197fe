"""The order network (reference ``DQNBPP`` with ``args.level == 'order'`` and ``bufferSize`` k > 1) and ``Agent.act``,
restated in torch from the equations of ``model.py`` -- TEST INFRASTRUCTURE: the checker of
``irbpp_b200.actor.DeviceOrderActor`` on machines without the reference, run in float64 on the device there.

The module has the reference's ``state_dict`` keys (those of the location network, ``oracle/dqn_port.py``, plus
``gat_project_layer`` and ``embedder``), so an order-level ``DQNBPP`` state dict loads into it and back.  What it
computes:

* ``model.py:184-189``  k item ids (``.long()`` truncates) and the 32 x 32 heightmap from column k on;
* ``model.py:361-363``  heightEncoder, 256 map features per bin;
* ``model.py:365-372``  the shape feature of each slot's item: the forward takes the per-shape features ``[S, 128]``
  (``DQNPort.shape_feature`` of each library shape's sampled points; the reference's index set is shared by the
  batch, so the feature depends on the shape only) and gathers them by id, ids clamped to ``[0, S)`` (the reference
  raises ``IndexError`` there);
* ``model.py:374-376``  gat_project_layer: ``[shape (128); map (256)]`` -> Linear(384,256), LeakyReLU, Linear(256,128);
* ``model.py:26-143, 145-171, 377-382``  one single-head graph-attention layer with nothing masked:
  ``h1 = h + W_out(softmax(Q K^T / sqrt(128)) V)``, ``h2 = h1 + Linear(ReLU(Linear(h1)))``, graph embedding the mean
  over the k slots;
* ``model.py:393-400``, ``agent.py:51-58``  the dueling heads over the slots, expected value, mask, argmax.
"""
import math

import torch
from torch import nn
from torch.nn import functional as F

from oracle.dqn_port import DQNPort, HM


class _Skip(nn.Module):
    """Holds ``module`` under the reference's key (``SkipConnection``, ``model.py:10-24``); the residual is applied
    in ``OrderDQNPort.embed``."""

    def __init__(self, module):
        super().__init__()
        self.module = module


class _Attention(nn.Module):
    """``MultiHeadAttention`` with one head, input and embedding width 128 (``model.py:26-65``)."""

    def __init__(self, dim=128):
        super().__init__()
        self.W_query = nn.Linear(dim, dim, bias=False)
        self.W_key = nn.Linear(dim, dim, bias=False)
        self.W_val = nn.Linear(dim, dim, bias=False)
        self.W_out = nn.Linear(dim, dim)
        with torch.no_grad():                       # model.py:61-65
            for p in self.parameters():
                p.uniform_(-1.0 / math.sqrt(p.size(-1)), 1.0 / math.sqrt(p.size(-1)))


class _Embedder(nn.Module):
    """``GraphAttentionEncoder(n_heads=1, embed_dim=128, n_layers=1)`` (``model.py:145-171``), by its keys."""

    def __init__(self, dim=128, ff=128):
        super().__init__()
        self.layers = nn.Sequential(nn.Sequential(_Skip(_Attention(dim)),
                                                  _Skip(nn.Sequential(nn.Linear(dim, ff), nn.ReLU(), nn.Linear(ff, dim)))))


class OrderDQNPort(DQNPort):
    """Order-level DQNBPP forward; ``forward(obs, shape_features)`` returns the atom probabilities ``[B, k, atoms]``
    for observations ``[B, k + 1024]``, ``shape_features`` being ``[S, 128]``, one row per library shape."""

    def __init__(self, buffer_size=10, atoms=31, hidden_size=128, noisy_std=0.5):
        super().__init__(selected_action=buffer_size, atoms=atoms, hidden_size=hidden_size, noisy_std=noisy_std)
        self.k = buffer_size
        self.gat_project_layer = nn.Sequential(nn.Linear(384, 256), nn.LeakyReLU(), nn.Linear(256, 128))
        self.embedder = _Embedder()

    def decode(self, obs):
        B, k = obs.shape[0], self.k
        return obs[:, :k].long(), obs[:, k:k + HM * HM].reshape(B, 1, HM, HM)

    def embed(self, obs, shape_features):
        """Slot embeddings ``h2`` ``[B, k, 128]`` and the graph embedding (their mean over the slots)."""
        ids, hm = self.decode(obs)
        B, k = ids.shape
        map_feature = self.heightEncoder(hm).reshape(B, -1)
        f = shape_features[ids.clamp(0, shape_features.shape[0] - 1)]
        h = self.gat_project_layer(torch.cat((f, map_feature[:, None, :].expand(B, k, 256)), dim=2))
        att = self.embedder.layers[0][0].module
        compat = (1.0 / math.sqrt(h.shape[2])) * torch.matmul(att.W_query(h), att.W_key(h).transpose(1, 2))
        h1 = h + att.W_out(torch.matmul(torch.softmax(compat, dim=-1), att.W_val(h)))
        h2 = h1 + self.embedder.layers[0][1].module(h1)
        return h2, h2.mean(1)
