"""The location network (reference ``DQNBPP`` with ``bufferSize == 1``) and ``Agent.act``, restated in torch from the
equations of ``model.py`` -- TEST INFRASTRUCTURE: the checker of ``irbpp_b200.actor`` on machines without the
reference, run in float64 on the device there.

The module has the reference's ``state_dict`` keys (42 of them, noise buffers included), so a ``DQNBPP`` state dict
loads into it and back.  What it computes:

* ``model.py:174-182``  candidate rows ``[rot, x, y, H]`` and the mask (column 4) of the first ``sel * 5`` values, the
  32 x 32 heightmap from ``sel * 5 + 9`` on;
* ``model.py:258-264``  heightEncoder: conv 1->16 k4 s2 p1, conv 16->32 k4 s2 p1, conv 32->4 k3 s1 p1, each followed by
  LeakyReLU, flattened (C, H, W) to 256;
* ``model.py:266-270, 334-335`` shapeEncoder (Linear 3->128, LeakyReLU, Linear 128->128, LeakyReLU, max over points),
  used only by ``shape_feature`` -- the forward takes the feature as an input;
* ``model.py:272-280, 337-342`` candidate embedding 4->32 LeakyReLU ->128, concat (shape | map | candidate), project
  512->256 LeakyReLU ->128;
* ``model.py:347-350`` rows with mask != 1 zeroed, graph embedding = mean over all ``sel`` rows;
* ``model.py:192-228, 393-400`` NoisyLinear value / advantage streams (train: mu + sigma * epsilon, eval: mu),
  ``q = v + a - mean_rows(a)``, softmax over the atoms;
* ``agent.py:51-58`` expected value over the support, ``-inf`` where ``mask != 1``, argmax over the rows.
"""
import math

import torch
from torch import nn
from torch.nn import functional as F

HM = 32
NOISY = ("fc_h_v", "fc_z_v", "fc_h_a", "fc_z_a")


class NoisyLinearPort(nn.Module):
    """Factorised-Gaussian noisy linear layer (model.py:192-228): same parameters, buffers and initialisation rule."""

    def __init__(self, in_features, out_features, std_init=0.5):
        super().__init__()
        self.in_features, self.out_features, self.std_init = in_features, out_features, std_init
        self.weight_mu = nn.Parameter(torch.empty(out_features, in_features))
        self.weight_sigma = nn.Parameter(torch.empty(out_features, in_features))
        self.register_buffer("weight_epsilon", torch.empty(out_features, in_features))
        self.bias_mu = nn.Parameter(torch.empty(out_features))
        self.bias_sigma = nn.Parameter(torch.empty(out_features))
        self.register_buffer("bias_epsilon", torch.empty(out_features))
        r = 1.0 / math.sqrt(in_features)
        with torch.no_grad():
            self.weight_mu.uniform_(-r, r)
            self.weight_sigma.fill_(std_init / math.sqrt(in_features))
            self.bias_mu.uniform_(-r, r)
            self.bias_sigma.fill_(std_init / math.sqrt(out_features))
        self.reset_noise()

    @staticmethod
    def _noise(n):
        x = torch.randn(n)
        return x.sign() * x.abs().sqrt()

    def reset_noise(self):
        e_in, e_out = self._noise(self.in_features), self._noise(self.out_features)
        self.weight_epsilon.copy_(torch.outer(e_out, e_in))
        self.bias_epsilon.copy_(e_out)

    def effective(self):
        if self.training:
            return self.weight_mu + self.weight_sigma * self.weight_epsilon, self.bias_mu + self.bias_sigma * self.bias_epsilon
        return self.weight_mu, self.bias_mu

    def forward(self, x):
        w, b = self.effective()
        return F.linear(x, w, b)


class DQNPort(nn.Module):
    """Location-level DQNBPP forward; ``forward(obs, shape_feature)`` returns the atom probabilities
    ``[B, sel, atoms]`` for observations of ``sel`` candidate rows."""

    def __init__(self, selected_action=500, atoms=31, hidden_size=128, noisy_std=0.5):
        super().__init__()
        self.sel, self.atoms = selected_action, atoms
        self.heightEncoder = nn.Sequential()
        self.heightEncoder.add_module("conv1", nn.Conv2d(1, 16, 4, stride=2, padding=1))
        self.heightEncoder.add_module("relu1", nn.LeakyReLU())
        self.heightEncoder.add_module("conv2", nn.Conv2d(16, 32, 4, stride=2, padding=1))
        self.heightEncoder.add_module("relu2", nn.LeakyReLU())
        self.heightEncoder.add_module("conv3", nn.Conv2d(32, 4, 3, stride=1, padding=1))
        self.heightEncoder.add_module("relu3", nn.LeakyReLU())
        self.shapeEncoder = nn.Sequential()
        self.shapeEncoder.add_module("linear1", nn.Linear(3, 128))
        self.shapeEncoder.add_module("relu1", nn.LeakyReLU())
        self.shapeEncoder.add_module("linear2", nn.Linear(128, 128))
        self.shapeEncoder.add_module("relu2", nn.LeakyReLU())
        self.init_candidate_embed = nn.Sequential(nn.Linear(4, 32), nn.LeakyReLU(), nn.Linear(32, 128))
        self.project_layer = nn.Sequential(nn.Linear(512, 256), nn.LeakyReLU(), nn.Linear(256, 128))
        self.fc_h_v = NoisyLinearPort(128, hidden_size, noisy_std)
        self.fc_h_a = NoisyLinearPort(128, hidden_size, noisy_std)
        self.fc_z_v = NoisyLinearPort(hidden_size, atoms, noisy_std)
        self.fc_z_a = NoisyLinearPort(hidden_size, atoms, noisy_std)

    def reset_noise(self):
        for name in NOISY:
            getattr(self, name).reset_noise()

    def shape_feature(self, points):
        """max over the points of shapeEncoder(points [B, n, 3]) (model.py:334-335)."""
        return self.shapeEncoder(points).max(dim=1)[0]

    def decode(self, obs):
        B, sel = obs.shape[0], self.sel
        rows = obs[:, :sel * 5].reshape(B, sel, 5)
        return rows[:, :, :4], rows[:, :, 4], obs[:, sel * 5 + 9:sel * 5 + 9 + HM * HM].reshape(B, 1, HM, HM)

    def embed(self, obs, shape_feature):
        """Row embeddings (zeroed where mask != 1) and the graph embedding (model.py:316-352)."""
        cand, mask, hm = self.decode(obs)
        B, sel = cand.shape[:2]
        map_feature = self.heightEncoder(hm).reshape(B, -1)
        x = torch.cat((shape_feature[:, None, :].expand(B, sel, 128), map_feature[:, None, :].expand(B, sel, 256),
                       self.init_candidate_embed(cand)), dim=2)
        e = self.project_layer(x)
        e = torch.where((mask != 1)[:, :, None], torch.zeros((), dtype=e.dtype, device=e.device), e)
        return e, e.mean(1)

    def advantage(self, e):
        return self.fc_z_a(F.relu(self.fc_h_a(e)))

    def forward(self, obs, shape_feature):
        e, g = self.embed(obs, shape_feature)
        v = self.fc_z_v(F.relu(self.fc_h_v(g)))[:, None, :]
        a = self.advantage(e)
        return F.softmax(v + a - a.mean(1, keepdim=True), dim=2)

    def sum_q(self, obs, shape_feature, support, mask=None):
        """agent.py:53-57: expected value per row, -inf where mask != 1."""
        s = (self.forward(obs, shape_feature) * support).sum(2)
        if mask is not None:
            s = s.masked_fill(mask != 1, -math.inf)
        return s

    def act(self, obs, shape_feature, support, mask=None):
        return self.sum_q(obs, shape_feature, support, mask).argmax(1)
