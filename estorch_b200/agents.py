"""Agent protocol.

Reference protocol (estorch.py:182,200 / :405,428,439): an object with
``rollout(policy) -> float`` (ES) or ``-> (float, bc: 1-D array)`` (NS family).
Arbitrary Python rollouts cannot run inside a kernel, so the device path needs
an agent that *declares* its computation:

``DeviceAgent`` -- rollout is "run the policy over a fixed observation batch
and reduce": ``return = -mean((policy(obs) - target)**2)`` (``loss="mse"``) or the
soft-target cross-entropy ``return = mean_b sum_c target_bc * log_softmax(policy(obs))_bc``
(``loss="cross_entropy"``: the policy's output is the logits) and (NS family)
``bc = policy(obs[:bc_obs]).flatten()[:bc_dim]`` (the 256-float behaviour
characteristic shape of examples/nsra_es.py:45-49).  It still implements the
reference protocol (``rollout``) with plain torch, so the very same object
runs under the CPU reference -- that is how the goldens and the CPU baseline
are produced.

``DeviceAgent(..., batch_size=B)`` holds a whole dataset and evaluates each generation on a fresh minibatch of
B rows of it, drawn on the device (``batches.batch_indices`` states which rows).

Any other agent (a gym loop, ...) is a *host agent*: the engine materialises
each member's parameter row on the device and calls ``rollout`` on the host,
exactly like estorch.py:195-202.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch

from .batches import batch_indices


LOSSES = ("mse", "cross_entropy")


class DeviceAgent:
    """Batch-regression or batch-classification agent evaluated by the fused CUDA kernel.

    ``loss="mse"`` (default): the return is minus the mean squared error against ``target``.
    ``loss="cross_entropy"``: ``target`` is ``[B, C]`` class weights per observation (one-hot or
    soft labels, finite and >= 0) and the return is minus the mean over the batch of the
    cross-entropy between those weights and the softmax of the policy's output.

    ``batch_size=B``: ``obs`` / ``target`` are a whole dataset of N rows (``dataset_obs`` / ``dataset_target``)
    and every generation is scored on a minibatch of B of them, the same minibatch for every member.
    Minibatch g takes positions g*B .. g*B + B - 1 of a stream of per-epoch permutations of the rows keyed by
    ``batch_seed`` (``batch_indices``), so each epoch visits every row once.  ``obs`` / ``target`` hold the
    current minibatch: batch 0 after construction, batch g after ``set_generation(g)``.  In fused mode ``ES``
    gathers each generation's minibatch on the device (the host copy is not updated); in hooks mode it calls
    ``set_generation`` before every generation.  ``rollout`` scores the current minibatch, and under the
    unmodified reference nothing advances it.  A behaviour characteristic needs fixed inputs, so
    ``batch_size`` with ``bc_obs`` / ``bc_dim`` is refused."""

    batch_size = None
    batch_seed = 0
    dataset_obs = dataset_target = None

    def __init__(self, obs: torch.Tensor, target: torch.Tensor, bc_obs: int = 0, bc_dim: int = 0, *,
                 loss: str = "mse", batch_size: Optional[int] = None, batch_seed: int = 0):
        if obs.dim() < 2 or target.dim() != 2 or obs.shape[0] != target.shape[0]:
            raise ValueError("obs must be [B, in] (or [B, C, H, W] for conv policies) and target [B, out]")
        if loss not in LOSSES:
            raise ValueError(f"loss must be one of {LOSSES}, got {loss!r}")
        if batch_size is not None:      # before the dataset is copied
            _check_batches(obs.shape[0], batch_size, bc_obs, bc_dim)
        self.obs = obs.detach().to(torch.float32).contiguous()
        self.target = target.detach().to(torch.float32).contiguous()
        if loss == "cross_entropy" and not (target.is_floating_point() and bool(torch.isfinite(self.target).all())
                                            and bool((self.target >= 0).all())):
            raise ValueError("loss='cross_entropy' needs target class weights that are finite and >= 0")
        self.loss = loss
        self.bc_obs = int(bc_obs)
        self.bc_dim = int(bc_dim)
        if bool(self.bc_obs) != bool(self.bc_dim):
            raise ValueError("bc_obs and bc_dim must both be zero or both be positive")
        if batch_size is not None:
            self._init_batches(batch_size, batch_seed)

    # -- minibatches of a dataset ---------------------------------------------
    def _init_batches(self, batch_size, batch_seed):
        self.batch_size, self.batch_seed = int(batch_size), int(batch_seed)
        self.dataset_obs, self.dataset_target = self.obs, self.target
        self.set_generation(0)

    def set_generation(self, generation: int):
        """Make ``obs`` / ``target`` minibatch ``generation`` of the dataset (``batch_size`` agents only)."""
        if self.batch_size is None:
            raise ValueError("set_generation needs an agent constructed with batch_size")
        idx = torch.from_numpy(batch_indices(self.batch_seed, generation, self.dataset_obs.shape[0],
                                             self.batch_size))
        self.obs, self.target = self.dataset_obs[idx], self.dataset_target[idx]

    # -- reference protocol (host / torch) ---------------------------------
    def rollout(self, policy):
        with torch.no_grad():
            p = next(policy.parameters())
            out = policy(self.obs.to(p.device))
            tgt = self.target.to(p.device)
            if self.loss == "cross_entropy":
                reward = float((tgt * torch.log_softmax(out, 1)).sum(1).mean())
            else:
                reward = float(-((out - tgt) ** 2).mean())
            if self.bc_dim:
                bc = out[:self.bc_obs].flatten()[:self.bc_dim].detach().cpu().numpy().copy()
                return reward, bc
        return reward

    # -- device protocol ------------------------------------------------------
    def next_batch(self, step: int) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
        """Called once per generation before evaluation.  Return ``None`` to keep
        the current batch, or ``(obs, target)`` host tensors (ideally pinned) of
        the same shapes to upload for this generation."""
        return None


def _check_batches(n, batch_size, bc_obs, bc_dim):
    """The rules of ``batch_size`` for a dataset of ``n`` rows."""
    if isinstance(batch_size, bool) or not isinstance(batch_size, (int, np.integer)) or not 1 <= batch_size <= n:
        raise ValueError(f"batch_size must be an int in [1, {n}] (the dataset's rows), got {batch_size!r}")
    if n >= 1 << 31:
        raise ValueError(f"a dataset of {n} rows is too large for minibatches (at most 2^31 - 1 rows)")
    if bc_obs or bc_dim:
        raise ValueError("batch_size cannot be combined with bc_obs / bc_dim: a behaviour characteristic needs "
                         "fixed inputs")


class SequenceAgent(DeviceAgent):
    """A fixed batch of sequences for a recurrent policy, evaluated by the fused CUDA kernel.

    ``obs`` is ``[B, T, in]`` and ``target`` ``[B, T, out]``.  Every sequence starts from the zero state; at
    step t the policy sees ``obs[:, t]`` and the state it returned at step t - 1.  The return scores all B*T
    steps as ``DeviceAgent`` scores its batch: ``loss="mse"`` is minus the mean squared error over every
    step and output, ``loss="cross_entropy"`` minus the mean over the B*T steps of each step's cross-entropy
    (its target row holds class weights).  A step whose cross-entropy target row is all zeros contributes 0,
    so a task can score only some steps, e.g. the last one.  The behaviour characteristic (NS family) is the
    outputs of the first ``bc_obs`` sequences, flattened in (b, t, out) order, then ``[:bc_dim]``.

    The policy is one ``nn.GRUCell`` or ``nn.LSTMCell``, one ``nn.Linear`` head and optionally a Tanh output,
    whose ``forward(x, state=None)`` returns ``(y, new_state)`` (see ``PopulationAgent``); with Adam and no
    overridden hook ``ES`` evaluates every perturbed member over the whole batch in one fused launch."""

    def __init__(self, obs: torch.Tensor, target: torch.Tensor, bc_obs: int = 0, bc_dim: int = 0, *,
                 loss: str = "mse", batch_size: Optional[int] = None, batch_seed: int = 0):
        if obs.dim() != 3 or target.dim() != 3 or tuple(obs.shape[:2]) != tuple(target.shape[:2]) or \
                obs.shape[1] < 1:
            raise ValueError("obs must be [B, T, in] and target [B, T, out] with the same B and T >= 1")
        if batch_size is not None:
            _check_batches(obs.shape[0], batch_size, bc_obs, bc_dim)
        super().__init__(obs.reshape(obs.shape[0], -1), target.reshape(target.shape[0], -1), bc_obs, bc_dim,
                         loss=loss)
        self.obs = self.obs.reshape(obs.shape)
        self.target = self.target.reshape(target.shape)
        if batch_size is not None:      # ``obs`` / ``target`` are a dataset of N sequences: minibatches of them
            self._init_batches(batch_size, batch_seed)

    def rollout(self, policy):
        with torch.no_grad():
            p = next(policy.parameters())
            obs, tgt = self.obs.to(p.device), self.target.to(p.device)
            state, ys = None, []
            for t in range(obs.shape[1]):
                # state None: policy(x), which is forward(x, state=None) for a recurrent policy
                res = policy(obs[:, t]) if state is None else policy(obs[:, t], state)
                if isinstance(res, tuple):
                    y, state = res
                else:                           # a memoryless policy: y only, and the state stays None
                    y = res
                ys.append(y)
            out = torch.stack(ys, 1)            # [B, T, out]
            if self.loss == "cross_entropy":
                reward = float((tgt * torch.log_softmax(out, 2)).sum(2).mean())
            else:
                reward = float(-((out - tgt) ** 2).mean())
            if self.bc_dim:
                bc = out[:self.bc_obs].flatten()[:self.bc_dim].detach().cpu().numpy().copy()
                return reward, bc
        return reward


class PopulationAgent:
    """An environment agent that steps one environment per population member, all members at once.

    Subclasses implement ``rollout_population(act, members)``, which runs ``members`` episodes side by
    side (environment state, done masks and termination are the agent's own) and returns
    ``returns[members]``; for the NS family it returns ``(returns[members], bc[members, bc_dim])`` and the
    subclass declares ``bc_dim`` (a positive int) as an attribute.

    ``act(obs)`` takes a float32 tensor on ``self.device``, shaped ``[members, in]`` or
    ``[members, B, in]``, and returns the policy outputs, ``[members, out]`` or ``[members, B, out]``.
    For the conv + VirtualBatchNorm policy of the reference's Atari example the observations are stacks of
    frames, ``[members, 4, 84, 84]`` or ``[members, B, 4, 84, 84]``, and the outputs ``[members, A]`` or
    ``[members, B, A]``; the members' VBN statistics over the policy's ``xref`` are computed once when
    ``act`` is built (they depend only on the weights), not on every call as the reference's forward does.
    Under ``ES`` in population mode, rows ``< members/2`` are the + members of the local antithetic pairs
    in pair order and the rest are their mirrors, and every row is evaluated by one fused CUDA launch of
    every perturbed policy; ``members == 1`` is the unperturbed policy.  ``act`` never synchronises with
    the device, so an episode loop that keeps its state on the device runs without host round trips.

    A recurrent policy -- one ``nn.GRUCell`` or ``nn.LSTMCell``, one ``nn.Linear`` head and optionally a Tanh
    output, whose ``forward(x, state=None)`` returns ``(y, new_state)`` -- is stepped with
    ``act(obs, state=None) -> (out, new_state)``.  ``state`` is h, ``[members, H]`` or ``[members, B, H]``
    (GRU), or the pair (h, c) of those (LSTM), in the same member order as ``obs``; None means zeros, as in
    torch.  In population mode one fused launch computes every member's cell step and head; the returned
    state is the next call's ``state``, and the agent owns it (resetting it where an episode ends, say).

    ``rollout(policy)`` -- the reference protocol -- is ``rollout_population`` with ``members == 1`` and
    ``act = policy`` (with the state passed through for a recurrent policy), so the same object also runs
    in hooks mode and under the reference itself.
    ``device`` is where the agent creates its tensors; ``ES`` sets it to the engine's device in
    population mode and to the policy's device otherwise."""

    device = torch.device("cpu")
    bc_dim = 0

    def rollout_population(self, act, members: int):
        raise NotImplementedError

    def rollout(self, policy):
        p = next(policy.parameters())

        def act(o, *state):
            if not state:                       # a memoryless policy: policy(obs)
                return policy(o.to(p.device)).to(o.device)
            y, s = policy(o.to(p.device), _state_to(state[0], p.device))
            return y.to(o.device), _state_to(s, o.device)
        with torch.no_grad():
            res = self.rollout_population(act, 1)
        if isinstance(res, tuple):
            ret, bc = res
            return float(torch.as_tensor(ret).reshape(-1)[0]), torch.as_tensor(bc).reshape(1, -1)[0].cpu().numpy().copy()
        return float(torch.as_tensor(res).reshape(-1)[0])


def _state_to(state, device):
    """A recurrent state (None, h, or a tuple (h, c)) moved to ``device``."""
    if state is None:
        return None
    if isinstance(state, (tuple, list)):
        return tuple(s.to(device) for s in state)
    return state.to(device)


SyntheticAgent = DeviceAgent
