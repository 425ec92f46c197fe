"""Glue between ``GpuVecEnv`` and the reference's learner for large N (SURVEY.md 8(f)2).

The reference's actor loop (``trainer.py:157-186``) is written for a handful of environments: per step it walks
``infos`` in Python (``:167-178``), appends to one ``ReplayMemory`` per environment in Python (``:183-185``) and
``Agent.learn`` samples ``int(batch_size / len(memory))`` transitions from EVERY memory (``agent.py:69``), which is
0 once there are more environments than batch entries.  At 4096 bins those loops, not the environment, set the
iteration rate.  This module keeps the loop's shape and removes the per-environment Python work:

* ``get_mask_from_state``  -- ``tools.get_mask_from_state`` (``tools.py:283-300``, selectedAction branch) as a view
  of the device observation;
* ``EpisodeStats``         -- the ``episode_rewards / episode_ratio / episode_counter`` deques of
  ``trainer.py:145-147,167-178`` fed from the step's result arrays (``LazyInfos.finished()``), no loop over bins;
* ``ReplayBank``           -- the N per-environment ring buffers of ``main.py:61-63`` as ONE device-resident bank
  ``[capacity, N, obs_len]``; ``append_batch`` replaces the loop of ``trainer.py:183-185``; ``sample`` draws a batch
  with the reference's segment rule made safe for N > batch_size (``segment_size``);
* ``segment_size``         -- the shim for ``agent.py:69``;
* ``PrioritizedReplayBank`` -- the reference's replay itself (``memory.py``: float32 sum tree, n-step returns,
  importance weights, stratified draws) for N memories on the device (``csrc/irbpp_replay.cuh``).
* ``device_learn``         -- ``Agent.learn`` (``agent.py:68-125``) with its two no-grad passes on the device
  (``DeviceActor.act`` / ``.target``) and, with ``gradient="device"``, the gradient pass's network and its backward
  at either level (``DeviceActor.log_prob`` / ``DeviceOrderActor.log_prob``); the optimiser stays in torch.

``ReplayBank`` samples uniformly; it exists so that the actor loop can be run end to end at N = 4096 and timed
(``tools/actor_loop.py``).
"""
from collections import deque

import numpy as np


def get_mask_from_state(state, selected_action):
    """Action mask = column 4 of the candidate rows (reference ``tools.py:298-299``); ``state`` is the
    ``[N, obs_len]`` observation (device tensor or NumPy array), the result a view ``[N, selected_action]``."""
    n = state.shape[0]
    return state[:, :selected_action * 5].reshape(n, selected_action, 5)[:, :, 4]


def segment_size(batch_size, num_memories):
    """``agent.py:69`` computes ``int(batch_size / len(memory))`` transitions per memory, 0 for more memories than
    batch entries.  Returns ``(memories_to_sample, per_memory)``: every memory when they fit, else ``batch_size``
    randomly chosen memories with one transition each."""
    per = batch_size // num_memories
    if per >= 1:
        return num_memories, per
    return batch_size, 1


class EpisodeStats(object):
    """The three ``deque(maxlen=10)`` of ``trainer.py:145-147`` updated from a step's ``(done, infos)`` without a
    Python loop over the bins that did not finish (``trainer.py:167-178`` touches every bin)."""

    def __init__(self, maxlen=10):
        self.episode_rewards = deque(maxlen=maxlen)
        self.episode_ratio = deque(maxlen=maxlen)
        self.episode_counter = deque(maxlen=maxlen)
        self.episodes = 0

    def update(self, done, infos):
        idx, ep_r, ratio, counter, valid = infos.finished()
        if len(idx):                                   # finished episodes of this step only (in bin order, as the reference)
            keep = valid.astype(bool)
            tail = slice(-self.episode_rewards.maxlen, None)      # only the last maxlen can survive in the deques
            self.episode_rewards.extend(ep_r[keep][tail].tolist())
            self.episode_ratio.extend(ratio[keep][tail].tolist())
            self.episode_counter.extend(counter[keep][tail].tolist())
        self.episodes += int(len(idx))
        return infos.valid_array()


class ReplayBank(object):
    """One ring buffer for all N environments on the device: slot ``t mod capacity`` holds the transition every
    environment made at its step ``t`` (the reference keeps ``N`` ``ReplayMemory`` objects of capacity
    ``memory_capacity / N`` each, ``main.py:61-63``).  Invalid samples (``infos[i]['Valid'] == False``,
    ``trainer.py:183-185``) are stored with weight 0 and never sampled."""

    def __init__(self, num_envs, capacity_per_env, obs_len, device, state_dtype=None):
        import torch
        self._torch = torch
        self.n, self.cap, self.device = int(num_envs), int(capacity_per_env), torch.device(device)
        self.states = torch.empty((self.cap, self.n, obs_len), dtype=state_dtype or torch.float32, device=self.device)
        self.actions = torch.zeros((self.cap, self.n), dtype=torch.int64, device=self.device)
        self.rewards = torch.zeros((self.cap, self.n), dtype=torch.float32, device=self.device)
        self.nonterminal = torch.zeros((self.cap, self.n), dtype=torch.bool, device=self.device)
        self.valid = torch.zeros((self.cap, self.n), dtype=torch.bool, device=self.device)
        self.t = 0

    def __len__(self):
        return min(self.t, self.cap)

    def append_from_env(self, env, state, action, reward_clip=0.0):
        """The same append with the step's reward / done / valid taken from the environment's DEVICE result arrays
        (``GpuVecEnv.last_step_device``): no host round trip, five device-to-device copies."""
        torch = self._torch
        dv = env.last_step_device()
        s = self.t % self.cap
        self.states[s].copy_(state)
        self.actions[s].copy_(action.reshape(-1))
        if reward_clip > 0:
            torch.clamp(dv["reward"], -reward_clip, reward_clip, out=self.rewards[s])       # trainer.py:180-181
        else:
            self.rewards[s].copy_(dv["reward"])
        torch.eq(dv["done"], 0, out=self.nonterminal[s])
        torch.ne(dv["valid"], 0, out=self.valid[s])
        self.t += 1

    def append_batch(self, state, action, reward, done, valid=None):
        """``self.mem[i].append(state[i], action[i], reward[i], done[i])`` for every i (``trainer.py:183-185``) as
        five batched copies.  ``reward`` / ``done`` / ``valid`` may be host arrays (what ``envs.step`` returns)."""
        torch = self._torch
        s = self.t % self.cap
        self.states[s].copy_(state)
        self.actions[s].copy_(torch.as_tensor(action).reshape(-1).to(self.device, non_blocking=True))
        self.rewards[s].copy_(torch.as_tensor(reward).reshape(-1).to(self.device, non_blocking=True))
        self.nonterminal[s].copy_(~torch.as_tensor(np.asarray(done)).to(self.device, non_blocking=True))
        if valid is None:
            self.valid[s].fill_(True)
        else:
            self.valid[s].copy_(torch.as_tensor(np.asarray(valid)).to(self.device, non_blocking=True))
        self.t += 1

    def sample(self, batch_size, generator=None):
        """A batch drawn with the reference's segment rule (``agent.py:69-75``): ``per`` transitions from each of
        ``m`` memories (all of them when ``N <= batch_size``, else ``batch_size`` random ones).  Returns
        ``(env_idx, slot_idx, states, actions, rewards, next_states, nonterminals)``; next states are the
        following slot of the same environment (the newest slot is never drawn)."""
        torch = self._torch
        filled = len(self)
        if filled < 2:
            raise RuntimeError("not enough transitions")
        m, per = segment_size(batch_size, self.n)
        if m == self.n:
            envs = torch.arange(self.n, device=self.device).repeat_interleave(per)
        else:
            envs = torch.randperm(self.n, device=self.device, generator=generator)[:m]
        newest = (self.t - 1) % self.cap
        off = torch.randint(1, filled, (envs.numel(),), device=self.device, generator=generator)      # 1 .. filled-1 steps back
        slots = (newest - off) % self.cap
        nxt = (slots + 1) % self.cap
        return (envs, slots, self.states[slots, envs], self.actions[slots, envs], self.rewards[slots, envs],
                self.states[nxt, envs], self.nonterminal[slots, envs])


class PrioritizedReplayBank(object):
    """The reference's N ``ReplayMemory`` objects (``main.py:61-63``, ``memory.py:95-208``: prioritized, n-step, a
    float32 sum tree per memory) as one device-resident bank of ``num_envs`` memories of ``capacity_per_env``
    transitions, driven by the kernels of ``csrc/irbpp_replay.cuh``: one launch per append, per sample and per priority
    update, for all memories at once.  The trees, indices and sampled transitions equal ``memory.py``'s for the same
    uniforms (``oracle/replay_port.py``); the uniforms here come from a counter-based generator of ``seed``.

    Where the reference's ``_get_sample_from_segment`` loops until it finds a valid leaf (``memory.py:163-170``, forever
    when a stratum holds only the n slots behind the write index or zero priorities), a stratum here gives up after
    ``max_attempts`` descents and ``sample`` raises ``RuntimeError`` naming the memory."""

    def __init__(self, num_envs, capacity_per_env, obs_len, device, discount=0.99, multi_step=3, priority_weight=0.4,
                 priority_exponent=0.5, seed=0, max_attempts=1024):
        import ctypes
        import torch
        from . import _lib
        self._torch, self._ctypes, self._lib = torch, ctypes, _lib.load()
        self.n, self.cap, self.obs_len = int(num_envs), int(capacity_per_env), int(obs_len)
        self.device = torch.device(device)
        self.discount, self.multi_step = float(discount), int(multi_step)
        self.priority_weight, self.priority_exponent = float(priority_weight), float(priority_exponent)
        self.seed, self.max_attempts, self.calls = int(seed), int(max_attempts), 0
        M, C, dev = self.n, self.cap, self.device
        self.states = torch.zeros((M, C, self.obs_len), dtype=torch.float32, device=dev)
        self.timesteps = torch.zeros((M, C), dtype=torch.int32, device=dev)
        self.actions = torch.zeros((M, C), dtype=torch.int64, device=dev)
        self.rewards = torch.zeros((M, C), dtype=torch.float32, device=dev)
        self.nonterminals = torch.zeros((M, C), dtype=torch.uint8, device=dev)
        self.tree = torch.zeros((M, 2 * C - 1), dtype=torch.float32, device=dev)
        self.state = torch.zeros((M, 4), dtype=torch.int32, device=dev)      # irbpp_replay_state: index, full, t, max
        self._flags = torch.zeros(1, dtype=torch.int32, device=dev)          # error bits of sample / update
        self._flags_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        self._mem = _lib.IrbppReplayMemory(M, C, self.obs_len, *(t.data_ptr() for t in (
            self.states, self.timesteps, self.actions, self.rewards, self.nonterminals, self.tree, self.state)))
        self._all = torch.arange(M, dtype=torch.int32, device=dev)
        self._rows = {}                                                       # k -> memory id of every row
        self._rng = np.random.default_rng(self.seed)
        with torch.cuda.device(dev):
            self._call(self._lib.irbpp_replay_init(ctypes.byref(self._mem), self._stream()))

    def _stream(self):
        return self._ctypes.c_void_p(self._torch.cuda.current_stream(self.device).cuda_stream)

    def _call(self, rc):
        from . import _lib
        _lib.check(self._lib, None, rc)

    def anneal_priority_weight(self, increase):
        """``priority_weight = min(priority_weight + increase, 1)`` (trainer.py:197)."""
        self.priority_weight = min(self.priority_weight + increase, 1.0)

    def append_from_env(self, env, state, action, reward_clip=0.0):
        """``self.mem[i].append(state[i], action[i], reward[i], done[i])`` for every bin with ``info['Valid']``
        (``trainer.py:181-186``), with reward / done / valid read from the environment's DEVICE result arrays
        (``GpuVecEnv.last_step_device``): one launch, no host round trip."""
        dv = env.last_step_device()
        self._append(state, action, dv["reward"], dv["done"], dv["valid"], reward_clip)

    def append_batch(self, state, action, reward, done, valid=None, reward_clip=0.0):
        """The same append from host arrays (what ``envs.step`` returns); ``valid=None`` appends every memory."""
        torch, dev = self._torch, self.device
        reward = torch.as_tensor(np.asarray(reward, np.float32).reshape(-1)).to(dev, non_blocking=True)
        done = torch.as_tensor(np.asarray(done).reshape(-1).astype(np.uint8)).to(dev, non_blocking=True)
        if valid is not None:
            valid = torch.as_tensor(np.asarray(valid).reshape(-1).astype(np.uint8)).to(dev, non_blocking=True)
        self._append(state, action, reward, done, valid, reward_clip)

    def _append(self, state, action, reward, done, valid, reward_clip):
        torch = self._torch
        if state.shape[0] != self.n or state.shape[-1] != self.obs_len or state.stride(-1) != 1:
            raise ValueError("state must be [%d, %d] with unit column stride" % (self.n, self.obs_len))
        state = state.to(self.device, torch.float32)
        action = torch.as_tensor(action).reshape(-1).to(self.device, torch.int64).contiguous()
        self._keep = (state, action, reward, done, valid)         # alive until the launch has read them
        with torch.cuda.device(self.device):
            self._call(self._lib.irbpp_replay_append(
                self._ctypes.byref(self._mem), state.data_ptr(), state.stride(0), action.data_ptr(), reward.data_ptr(),
                done.data_ptr(), valid.data_ptr() if valid is not None else None, float(reward_clip), self._stream()))

    def sample(self, batch_size, uniforms=None):
        """``Agent.learn``'s batch (``agent.py:69-82``): ``(tree_idxs, states, actions, returns, next_states,
        nonterminals [B, 1], weights, mem_ids)``, memory by memory as ``torch.cat`` orders it.

        With ``N <= batch_size`` every memory gives ``batch_size // N`` samples, as the reference does.  With
        ``N > batch_size`` (where ``int(batch_size / N)`` is 0 and the reference stops) ``batch_size`` distinct memories
        give one sample each (``segment_size``); under the reference's per-memory normalisation a single sample is its
        memory's batch maximum, so every weight is then exactly 1.

        The call reads one 4-byte error word back through pinned memory, which synchronises the current stream once:
        a starved stratum or an out-of-range row of an earlier ``update_priorities`` raises here, before the batch can
        be used.  ``uniforms`` (float64 [rows, attempts] on the device) replaces the generator, for parity tests."""
        torch, ct = self._torch, self._ctypes
        G, k = segment_size(batch_size, self.n)
        if G == self.n:
            ids = self._all
        else:
            pick = self._rng.choice(self.n, G, replace=False).astype(np.int32)
            ids = torch.from_numpy(pick).pin_memory().to(self.device, non_blocking=True)
        return self._sample(ids, k, uniforms)

    def _sample(self, ids, k, uniforms=None):
        torch, ct, dev = self._torch, self._ctypes, self.device
        B, L = ids.numel() * k, self.obs_len
        out = dict(tree_idx=torch.empty(B, dtype=torch.int64, device=dev),
                   states=torch.empty((B, L), dtype=torch.float32, device=dev),
                   actions=torch.empty(B, dtype=torch.int64, device=dev),
                   returns=torch.empty(B, dtype=torch.float32, device=dev),
                   next_states=torch.empty((B, L), dtype=torch.float32, device=dev),
                   nonterminals=torch.empty(B, dtype=torch.float32, device=dev),
                   weights=torch.empty(B, dtype=torch.float32, device=dev),
                   attempts=torch.empty(B, dtype=torch.int32, device=dev),
                   error=torch.empty(B, dtype=torch.int32, device=dev))
        from . import _lib
        batch = _lib.IrbppReplayBatch(*(out[n].data_ptr() for n in (
            "tree_idx", "states", "actions", "returns", "next_states", "nonterminals", "weights", "attempts", "error")))
        attempts = self.max_attempts if uniforms is None else int(uniforms.shape[1])
        with torch.cuda.device(dev):
            self._call(self._lib.irbpp_replay_sample(
                ct.byref(self._mem), ids.data_ptr(), ids.numel(), k, self.multi_step, self.discount, self.priority_weight,
                attempts, self.seed, self.calls, uniforms.data_ptr() if uniforms is not None else None, ct.byref(batch),
                self._flags.data_ptr(), self._stream()))
            self.calls += 1
            self._flags_host.copy_(self._flags, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
        flags = int(self._flags_host[0])
        if flags:
            self._flags.zero_()
            err = out["error"].cpu().numpy()
            mem_ids = ids.repeat_interleave(k).cpu().numpy()
            msg = []
            if flags & (1 << 1):
                msg.append("no valid transition in %d draws of a stratum of memory %s (too few transitions, or only "
                           "zero priorities)" % (attempts, sorted(set(mem_ids[err == 1].tolist()))))
            if flags & (1 << 2):
                msg.append("memory id out of range: %s" % sorted(set(mem_ids[err == 2].tolist())))
            if flags & (1 << 3):
                msg.append("an earlier update_priorities had a memory id or tree index out of range")
            raise RuntimeError("prioritized replay: " + "; ".join(msg))
        self.last_attempts, self.last_error = out["attempts"], out["error"]
        rows = ids if k == 1 else self._rows.get(k)
        if rows is None or ids is not self._all:
            rows = ids.repeat_interleave(k)
            if ids is self._all:
                self._rows[k] = rows
        return (out["tree_idx"], out["states"], out["actions"], out["returns"], out["next_states"],
                out["nonterminals"].reshape(B, 1), out["weights"], rows)

    def update_priorities(self, tree_idxs, mem_ids, loss):
        """``memory[i].update_priorities(idxs[i], loss[i * k:(i + 1) * k])`` for every memory (``agent.py:123-124``)
        as one launch on the device tensors: leaf ← loss ** priority_exponent, last row wins on a duplicated index."""
        torch = self._torch
        idx = tree_idxs.to(self.device, torch.int64).contiguous()
        mids = mem_ids.to(self.device, torch.int32).contiguous()
        loss = loss.detach().to(self.device, torch.float32).contiguous()
        self._keep_upd = (idx, mids, loss)
        with torch.cuda.device(self.device):
            self._call(self._lib.irbpp_replay_update_priorities(
                self._ctypes.byref(self._mem), mids.data_ptr(), idx.data_ptr(), loss.data_ptr(), idx.numel(),
                self.priority_exponent, self._flags.data_ptr(), self._stream()))


def device_learn(agent, bank, online_actor, target_actor, gradient="torch"):
    """``agent.learn(mem)`` (``agent.py:68-125``) on a ``PrioritizedReplayBank``, for either network level (the level
    follows from the actors): ``online_actor`` wraps ``agent.online_net`` and ``target_actor`` wraps
    ``agent.target_net`` (both ``DeviceActor`` or both ``DeviceOrderActor``, read live).  Returns the loss ``[B]`` on
    the device.  The calls keep the reference's order, so torch's RNG is consumed as the reference consumes it:

    1. ``bank.sample(agent.batch_size)``;
    2. ``agent.online_net(states, log=True)`` with gradients (agent.py:85-86);
    3. ``online_actor.act(next_states)``, unmasked: the double-Q a* (agent.py:90-92);
    4. ``agent.target_net.reset_noise()`` (agent.py:94);
    5. ``target_actor.target(...)``: p(s', a*; target) and its projection m (agent.py:96-115);
    6. the loss, the importance-weighted mean, ``backward``, ``clip_grad_norm_`` and ``optimiser.step()`` exactly as
       agent.py:117-121;
    7. ``bank.update_priorities`` with the loss (agent.py:123-124).

    ``gradient="device"`` replaces step 2 with ``online_actor.log_prob(states, actions)`` at either level: the
    candidate-row network (``DeviceActor``, ``irbpp_dqn_log_prob``) or the order network's per-slot layers and
    graph attention (``DeviceOrderActor``, ``irbpp_dqn_order_log_prob``) and their backward passes run as kernels,
    while the encoders, the NoisyLinear rebuild, the loss, ``clip_grad_norm_`` and Adam stay in torch.  An order actor
    given states of another width (a location-level batch) raises ``ValueError`` before it is called.
    ``gradient="torch"`` runs the module itself; it is the reference the device path is tested against.

    One difference from the reference: its three forward passes each draw point indices with ``np.random``
    (model.py:331, 367); here the device passes draw from the counter-based generator of their actors'
    ``DeviceShapeClouds`` / ``OrderShapeClouds``, one index set per pass (with ``gradient="torch"`` the gradient pass
    draws as the module does)."""
    import torch
    from torch.nn.utils import clip_grad_norm_
    if gradient not in ("torch", "device"):
        raise ValueError("gradient must be 'torch' or 'device', got %r" % (gradient,))
    if gradient == "device" and not callable(getattr(online_actor, "log_prob", None)):
        raise ValueError("gradient='device' supports the location level (DeviceActor.log_prob) and the order level "
                         "(DeviceOrderActor.log_prob); %s has no log_prob" % type(online_actor).__name__)
    idxs, states, actions, returns, next_states, nonterminals, weights, mem_ids = bank.sample(agent.batch_size)
    B = states.shape[0]
    if gradient == "device":
        _check_level(online_actor, states.shape[-1])
        log_ps_a = online_actor.log_prob(states, actions)
    else:
        log_ps = agent.online_net(states, log=True)
        log_ps_a = log_ps[torch.arange(B, device=log_ps.device), actions]
    with torch.no_grad():
        next_actions = online_actor.act(next_states)
        agent.target_net.reset_noise()
        m, _ = target_actor.target(next_states, next_actions, returns, nonterminals, agent.Vmin, agent.Vmax,
                                   agent.discount ** agent.n, with_p=False)
    loss = -torch.sum(m * log_ps_a, 1)
    agent.online_net.zero_grad()
    (weights * loss).mean().backward()
    clip_grad_norm_(agent.online_net.parameters(), agent.norm_clip)
    agent.optimiser.step()
    bank.update_priorities(idxs, mem_ids, loss.detach())
    return loss


def _check_level(online_actor, width):
    """``ValueError`` when a ``DeviceOrderActor`` is given observations of ``width`` values that are not the order
    level's ``bufferSize + 1024`` (2 <= bufferSize <= 32); a location actor checks its own states in ``log_prob``."""
    from .actor import HM, MAX_BUFFER, DeviceOrderActor
    if isinstance(online_actor, DeviceOrderActor) and not 2 <= width - HM * HM <= MAX_BUFFER:
        raise ValueError("the sampled states have %d values, not an order observation (bufferSize + 1024); a "
                         "location-level batch needs a DeviceActor" % width)
