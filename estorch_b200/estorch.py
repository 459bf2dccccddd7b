"""Host-side mirror of the reference's algorithm classes (estorch/estorch.py).

Same class names, constructor signatures, ``train`` / ``terminate`` / ``log``
API, overridable hooks and public attributes as the reference (SURVEY 8b), but
the body of a generation runs on the GPU through the C ABI in include/estk.h:

    reference (CPU, estorch.py)                 here (H100)
    -------------------------------------------  ------------------------------------------
    _sample_policy :187-193  fresh RNG + cats    noise-table offsets (estk_make_offsets)
    MPI Send/Recv of P x n rows :207-233         nothing to send: every rank regenerates rows
    _calculate_returns :195-202 (python loop)    estk_eval_mlp (fused) | host rollouts (plumbing)
    rank_transformation + torch.mm :174-179      estk_rank_grad[_adam] (+ one NCCL all-reduce)
    grad scatter/clamp :236-244, Adam.step :245  fused Adam epilogue (or torch optimizer.step)
    _after_optimize :181-185                     estk_eval_mlp (centre, offsets NULL) + estk_track_best

Three execution modes, chosen per instance:

* fused  -- DeviceAgent + recognised MLP policy + torch.optim.Adam + no hook
            overridden: a generation is a handful of kernel launches, nothing
            touches the host unless the user reads an attribute.
* population -- PopulationAgent (environments stepped by user code, one per
            member) + recognised MLP, conv + VirtualBatchNorm or recurrent
            (GRUCell / LSTMCell + Linear head) policy + Adam + no hook
            overridden, on one GPU: every environment step is one launch
            that evaluates every perturbed policy on its member's own observation
            (and state) (estk_eval_mlp / estk_eval_conv_vbn with ESTK_ACTIONS; the
            conv policy's VBN statistics are one more launch per generation); ranks,
            gradient and Adam as in fused mode.
* hooks  -- anything else (host agents such as gym loops, custom subclasses
            overriding ``_sample_policy`` / ``_calculate_grad`` / ..., other
            optimizers): the reference's own control flow through its hooks,
            with noise rows and the gradient still produced on the device.
"""
from __future__ import annotations

import copy
import os
import sys
import time
import weakref
from collections import OrderedDict
from enum import Enum
from typing import Optional

import numpy as np
import torch

from ._capi import ESTK_CONV_VBN_STATS_FLOATS, ESTK_LOSS_ACCURACY, ESTK_LOSS_XENT, ESTK_MAX_POPULATION
from .agents import DeviceAgent, PopulationAgent, SequenceAgent
from .backend import adam_desc, new_state, read_state, write_state
from .policy_spec import (CNNSpec, ConvVBNSpec, RNNSpec, cnn_spec_from_module, conv_vbn_spec_from_module,
                          mlp_spec_from_module, rnn_spec_from_module)
from .population import LazyPopulation, NoiseHandle

__all__ = ["ES", "NS_ES", "NSR_ES", "NSRA_ES", "rank_transformation"]

DEFAULT_NOISE_TABLE_SIZE = 1 << 28   # fp32 unit normals = 1 GiB per GPU (SURVEY 8d)
# Smallest sigma at which eval_precision="auto" evaluates an MLP in "f16".  f16 rounds each formed weight
# theta +- sigma*eps to 11 bits, about 2^-11 |theta|: once sigma*eps is not much larger than that, the
# antithetic differences that order the population turn to noise.  Measured on an H100 80GB HBM3 (700 W)
# against a float64 evaluate (tests/test_signal_fidelity_gpu.py, DESIGN.md 4.3): at sigma >= 0.02 the f16
# gradient is within 3e-2 (rel-L2) of the float64-return gradient for weights up to 8x their initial scale;
# at sigma = 5e-3 it reaches 3.3e-2 at 4x, at sigma = 1e-3 4.4e-2.  Below the threshold "auto" evaluates
# in fp32, whose ranks are the float64 ranks up to near-ties within fp32 rounding.
AUTO_F16_MIN_SIGMA = 0.02
_UNFUSED_ADAM_FLAGS = ("amsgrad", "maximize", "differentiable", "decoupled_weight_decay")


def _refuse_unfused_adam_flags(group):
    """The fused epilogue is torch's Adam with L2 weight decay only.  Constructor keywords that ask for
    something else select hooks mode (ES._decide_fused); switched on in ``param_groups`` after
    construction, they would silently give a different optimizer."""
    on = [k for k in _UNFUSED_ADAM_FLAGS if group.get(k)]
    if on:
        raise ValueError(f"the fused Adam step does not implement {', '.join(on)}; pass it to the optimizer's "
                         "constructor instead (hooks mode runs torch's own optimizer)")


# ----------------------------------------------------------------------------
# rank transform (public helper, estorch.py:15-39) -- host numpy; the device
# path computes the same quantity inside estk_rank_grad*.
# ----------------------------------------------------------------------------
def _compute_ranks(rewards):
    r = np.asarray(rewards).reshape(-1)
    ranks = np.empty(r.size, dtype=int)
    ranks[np.argsort(r, kind="stable")] = np.arange(r.size)
    return ranks


def rank_transformation(rewards):
    """Centred ranks in [-0.5, 0.5] (float64), lowest reward -> -0.5.

    >>> rank_transformation([-123, -50, 3, -5, 20, 10, 100])
    array([-0.5, -0.33333333, 0., -0.16666667, 0.33333333, 0.16666667, 0.5])
    Ties are broken by index (the reference leaves them unspecified).
    """
    ranks = _compute_ranks(rewards)
    size = ranks.size
    return (np.arange(size) / (size - 1) - 0.5)[ranks]


class _Algorithm(Enum):
    classic = 1
    novelty = 2


def _release_shm(shm, owner):
    try:
        shm.close()
        if owner:
            shm.unlink()
    except Exception:
        pass


_LIVE = weakref.WeakSet()      # instances that may hold CUDA graphs with captured collectives


_OWN_PROCESS_GROUP = False     # this module called init_process_group (then it also destroys it at exit)
_EXIT_HOOK = False


def _shutdown_dist():
    """Process exit of a multi-GPU rank.  A CUDA graph that captured NCCL kernels keeps a reference on
    the communicator, and destroying the communicator first never returns: graphs go first, then the mappings of the peers'
    workspaces, then -- if this module created it -- the process group.  A script that destroys the process group itself calls ``es.close()`` (or drops the
    instance) first."""
    import gc
    import torch.distributed as dist
    for es in list(_LIVE):
        es.__dict__.pop("_graphs", None)
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    for es in list(_LIVE):                # unmap the peers' workspaces; this process's own allocations are left to
        if hasattr(es._be, "peer_close_all"):   # process teardown (freeing them needs every peer to have unmapped
            es._be.peer_close_all()             # first, and a barrier in an exit hook would hang if a rank died)
    if dist.is_initialized() and _OWN_PROCESS_GROUP:
        dist.destroy_process_group()


_NVTX = os.environ.get("ESTORCH_B200_NVTX", "0") == "1"


def _nvtx_push(name):
    """Phase markers for nsys / ncu --nvtx (off unless ESTORCH_B200_NVTX=1; the reference has no tracing)."""
    if _NVTX:
        torch.cuda.nvtx.range_push(name)


def _nvtx_pop():
    if _NVTX:
        torch.cuda.nvtx.range_pop()


def _builtin(fn):
    fn._estk_builtin = True
    return fn


def _dist_env():
    """(rank, world, local_rank) of this process; one process per GPU."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size(), int(os.environ.get("LOCAL_RANK", dist.get_rank()))
    return (int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)),
            int(os.environ.get("LOCAL_RANK", 0)))


class _PolicySlot:
    """One (policy, optimizer) pair with device-resident flat state."""

    def __init__(self, module, optimizer, be, flatten: bool):
        self.module = module
        self.optimizer = optimizer
        self.be = be
        params = list(module.parameters())
        self.n = sum(p.numel() for p in params)
        self.theta = be.zeros(self.n)
        self.m = be.zeros(self.n)
        self.v = be.zeros(self.n)
        self.best_theta = be.zeros(self.n)
        self.theta_prev = be.zeros(self.n)     # centre of the last sampled population
        self.state = new_state(be.device)
        self.theta16 = None                    # bf16 shadow of theta (eval_precision="bf16s")
        self.flattened = flatten
        with torch.no_grad():
            self.theta.copy_(torch.nn.utils.parameters_to_vector(params).detach().to(be.device))
            if flatten:
                # parameters become views of the flat vector: the module always
                # shows the live theta, no per-generation copies
                idx = 0
                for p in params:
                    p.data = self.theta[idx: idx + p.numel()].view(p.shape)
                    idx += p.numel()

    def ensure_flat(self):
        """Re-establish parameter <-> flat-vector aliasing if user code re-pointed
        ``param.data`` (``torch.nn.utils.vector_to_parameters`` does exactly that)."""
        if not self.flattened:
            return
        idx, esz = 0, self.theta.element_size()
        with torch.no_grad():
            for p in self.module.parameters():
                sz = p.numel()
                if p.data.data_ptr() != self.theta.data_ptr() + idx * esz or p.device != self.theta.device:
                    self.theta[idx: idx + sz].copy_(p.data.reshape(-1))
                    p.data = self.theta[idx: idx + sz].view(p.shape)
                idx += sz

    def push_theta(self):
        """module -> flat (hooks mode: the torch optimizer updated the module)."""
        if not self.flattened:
            with torch.no_grad():
                self.theta.copy_(torch.nn.utils.parameters_to_vector(self.module.parameters())
                                 .detach().to(self.be.device))

    def mirror_adam_state(self):
        """Expose the fused Adam moments through the torch optimizer object."""
        if not self.flattened:
            return
        step = float(read_state(self.state)["adam_step"])
        idx = 0
        for p in self.module.parameters():
            sz = p.numel()
            self.optimizer.state[p] = {"step": torch.tensor(step),
                                       "exp_avg": self.m[idx: idx + sz].view(p.shape),
                                       "exp_avg_sq": self.v[idx: idx + sz].view(p.shape)}
            idx += sz


class ES:
    """Classic Evolution Strategy (OpenAI-ES, Salimans et al. 2017) with the
    constructor and training API of the reference ``estorch.ES``
    (estorch.py:68-308).

    Args (identical to the reference, estorch.py:121-123):
        policy: ``nn.Module`` *class*; instantiated as ``policy(**policy_kwargs)``.
        agent: class with ``rollout(policy) -> float``; ``agent(**agent_kwargs)``.
        optimizer: ``torch.optim`` class; ``optimizer(params, **optimizer_kwargs)``.
        population_size: total evaluations per generation (both mirrored halves).
        sigma: noise standard deviation.
        device: device of the modules handed to a *host* agent's ``rollout``.
    Engine options (keyword-only, all optional):
        noise_table_size: length of the shared unit-normal table (default 2**28).
        noise_seed: seed of the table and of the per-generation offsets.
        log_interval: call ``log()`` every k-th generation only (default 1 =
            reference behaviour).
        eval_precision: arithmetic of the fused evaluate kernel:
            ``"fp32"``  CUDA-core path, fp32 throughout;
            ``"f16"``   wgmma tensor cores with fp16 operands (11-bit significand, the
                        TF32 class) and fp32 accumulation; every weight is formed in fp32
                        from the fp32 theta and the (exactly 16-bit representable) noise
                        value and rounded once; observations enter as hi + lo halves.
                        On an MLP shape outside the cluster kernel's rule (widths not
                        multiples of 64 / 32 or above 512, B not a multiple of 256, e.g. a
                        10-class head or a 784-wide input) it selects ``"f16_any"``: the same
                        arithmetic per element on a streamed wgmma kernel, for any widths and
                        any batch (no folded post-update rollout there).
                        For the conv + VirtualBatchNorm policy (examples/atari.py) ``"f16"``
                        is an opt-in mma.sync kernel whose weights, inputs and normalised
                        activations all enter as hi + lo fp16 pairs (22-bit operands);
            ``"auto"``  (default) ``"f16"`` when the MLP shape supports it and ``sigma >=
                        AUTO_F16_MIN_SIGMA`` (0.02), else ``"fp32"`` (ReLU, Tanh, ELU, SiLU and
                        LeakyReLU MLPs alike, with the squared error, the cross-entropy or the accuracy
                        of ``DeviceAgent(loss=...)``; always ``"fp32"`` for the conv policy).
                        Accuracy of "f16" against a float64 evaluate, on what ES consumes (H100 at 700 W,
                        P = 64): at sigma >= 0.02 and weights up to 8x their initial scale the gradient
                        is within 3e-2 (rel-L2) of the float64-return gradient and the returns within
                        about 2e-4 (max-norm relative; 1e-5 only at init-scale weights).  Below, the
                        11-bit rounding of each formed weight, about 2^-11 |theta|, reorders members:
                        gradient error up to 3.3e-2 at sigma = 5e-3 and 4x init, 4.4e-2 at 1e-3, and at
                        sigma = 2e-4 up to a quarter of the antithetic differences change sign.  There
                        "auto" evaluates in fp32, whose ranks are the float64 ranks up to near-ties
                        within fp32 rounding; an explicit ``"f16"`` is still honoured;
            ``"bf16"`` / ``"bf16s"``  explicit opt-in, lower precision (8-bit significand;
                        ``bf16s`` additionally reads bf16 shadows of theta and the table);
                        MLP policies only;
            ``"tf32"``  explicit opt-in for fused convolutional policies (a Conv2d stack + Linear head
                        on a DeviceAgent, with or without ``batch_size``, ES and the NS family): every
                        layer an implicit GEMM on TF32 tensor cores (mma.sync), each formed fp32 weight
                        and each layer input rounded to nearest (ties away) to an 11-bit significand (the
                        TF32 class), fp32 accumulation, fp32 bias and activations
                        (include/estk_eval_cnn_tf32.h).  Every layer output up to 2**26 floats per image.
                        On one H100 80GB HBM3 at 700 W it evaluates 1.8x (MNIST shape), 9.9x (Atari
                        shape) and 3.4x (MinAtar shape) faster than "fp32" (DESIGN §9).  Accuracy against
                        a float64 evaluate, on what ES consumes (same card, P = 64): at sigma >= 5e-3 and
                        weights up to 8x their initial scale the gradient is within 1.8e-2 (rel-L2) of the
                        float64-return gradient; below, members reorder (4.2e-2 at sigma = 1e-3 and 4x
                        init, up to 0.33 at 2e-4).  Population mode stays fp32; MLP, conv +
                        VirtualBatchNorm and recurrent policies refuse it.
    Population size: any even value up to ``ESTK_MAX_POPULATION`` (2**22); larger values raise
    ``ValueError`` here.  Device memory that grows with P: the returns (4 B per member), ranks
    (4 B), offsets and evaluation order (12 B per pair), the library workspace (about 20 B per
    member beyond 32768, plus the evaluate partials, 4 B per member and observation chunk), and for
    the NS family the behaviour characteristics, ``P * bc_dim`` floats (1 GB at P = 2**20,
    bc_dim = 256).  Hooks mode (host agents) still rolls out one member at a time on the host.
    Attributes as documented at estorch.py:108-117.
    """

    _ALGORITHM_TYPE = _Algorithm.classic

    def __init__(self, policy, agent, optimizer, population_size, sigma=0.01,
                 device=torch.device("cpu"), policy_kwargs={}, agent_kwargs={},
                 optimizer_kwargs={}, *, noise_table_size=None, noise_seed=42,
                 log_interval=1, eval_precision="auto", _backend=None):
        self.rank, self.n_workers, self._local_rank = _dist_env()
        self.population_size = int(population_size)
        assert not (self.population_size % self.n_workers)           # estorch.py:130
        if self.population_size % 2 or self.population_size < 2:
            raise ValueError("population_size must be even (mirrored sampling, estorch.py:190)")
        if self.population_size > ESTK_MAX_POPULATION:
            raise ValueError(f"population_size {self.population_size} exceeds the engine's limit of "
                             f"{ESTK_MAX_POPULATION} members (ESTK_MAX_POPULATION)")
        if (self.population_size // 2) % self.n_workers:
            raise ValueError("population_size/2 antithetic pairs must divide evenly over the GPUs")
        self.device = torch.device(device)
        self.sigma = sigma
        self._stop = False
        self._trained = False
        self._noise_seed = int(noise_seed)
        self._log_interval = max(1, int(log_interval))
        self._policy_cls, self._policy_kwargs = policy, dict(policy_kwargs)
        self._optimizer_cls, self._optimizer_kwargs = optimizer, dict(optimizer_kwargs)

        if _backend is None:
            from .backend import CudaBackend       # raises loudly without a GPU / the .so
            _backend = CudaBackend(torch.device("cuda", self._local_rank % max(1, torch.cuda.device_count())))
        self._be = _backend
        self._dev = self._be.device

        self.agent = agent(**agent_kwargs)
        self._device_agent = isinstance(self.agent, DeviceAgent)
        obs_shape = getattr(self.agent, "obs_shape", None) if isinstance(self.agent, PopulationAgent) else None
        if obs_shape is not None and not (isinstance(obs_shape, (tuple, list)) and len(obs_shape) == 3 and all(
                isinstance(d, int) and not isinstance(d, bool) and d > 0 for d in obs_shape)):
            raise ValueError(f"PopulationAgent.obs_shape must be None or (c, h, w), three positive ints; got "
                             f"{obs_shape!r}")
        # a device agent with batch_size: every generation evaluates a fresh minibatch of its dataset
        self._sampling = self._device_agent and self.agent.batch_size is not None
        if self._sampling and type(self.agent).next_batch is not DeviceAgent.next_batch:
            raise ValueError("an agent with batch_size draws its minibatches on the device; it cannot also "
                             "override next_batch (one batch source per agent)")
        self.target = policy(**policy_kwargs).to(self.device)       # estorch.py:142
        parameters = torch.nn.utils.parameters_to_vector(self.target.parameters())
        self.n_parameters = parameters.shape[0]
        # the recurrent recogniser comes last and draws from a private generator only: the global RNG stream
        # that the other two leave behind is the one every policy saw before recurrent policies were recognised
        self._spec = (mlp_spec_from_module(self.target) or conv_vbn_spec_from_module(self.target)
                      or rnn_spec_from_module(self.target))
        # a Conv2d stack does not fix H and W: the CNN recogniser takes the shape of a device agent's images,
        # and comes after the other three for the same reason as the recurrent one
        if self._spec is None and type(self.agent) is not SequenceAgent and isinstance(self.agent, DeviceAgent) \
                and self.agent.obs.dim() == 4:
            self._spec = cnn_spec_from_module(self.target, tuple(self.agent.obs.shape[1:]))
        # ... and for a population agent, the shape of one observation it declares
        if self._spec is None and obs_shape is not None:
            self._spec = cnn_spec_from_module(self.target, tuple(obs_shape))
        self._is_conv = isinstance(self._spec, ConvVBNSpec)
        self._is_rnn = isinstance(self._spec, RNNSpec)
        self._is_cnn = isinstance(self._spec, CNNSpec)
        self._fused = self._decide_fused(optimizer)
        self._population = self._fused and isinstance(self.agent, PopulationAgent)
        if isinstance(self.agent, PopulationAgent):
            self.agent.device = self._dev if self._population else self.device
        self._host_cache = {}
        if eval_precision not in ("auto", "fp32", "f16", "bf16", "bf16s", "tf32"):
            raise ValueError("eval_precision must be 'auto', 'fp32', 'f16', 'bf16', 'bf16s' or 'tf32'")
        if self._population and eval_precision not in ("auto", "fp32"):
            raise ValueError("population mode (a PopulationAgent) computes every member's actions in fp32 only: "
                             "eval_precision must be 'auto' or 'fp32'")
        if self._fused and not self._is_cnn and eval_precision == "tf32":
            raise ValueError("eval_precision='tf32' is for convolutional policies (a Conv2d stack + Linear head "
                             "on a DeviceAgent); MLP, conv + VirtualBatchNorm and recurrent policies have no "
                             "'tf32' mode")
        if self._fused and self._is_rnn and eval_precision not in ("auto", "fp32"):
            raise ValueError("the recurrent sequence evaluate (a SequenceAgent) is fp32 only: "
                             "eval_precision must be 'auto' or 'fp32'")
        if self._fused and self._is_cnn and eval_precision not in ("auto", "fp32", "tf32"):
            raise ValueError("the convolutional evaluate (a Conv2d stack + Linear head) is fp32 only: "
                             "eval_precision must be 'auto' or 'fp32'")
        self._precision = "fp32"
        if self._fused and self._is_cnn and eval_precision == "tf32":
            B = self.agent.batch_size or self.agent.obs.shape[0]
            if not self._be.eval_supports_tf32_cnn(self._spec.dims, B, act=self._act_code()):
                raise ValueError("eval_precision='tf32' serves convolutional policies whose largest layer output "
                                 "is at most 2**26 floats per image")
            self._precision = "tf32"
        if self._fused and self._is_conv and eval_precision in ("bf16", "bf16s"):
            raise ValueError("the conv + VirtualBatchNorm evaluate kernel has 'fp32' and 'f16' modes only")
        if self._fused and self._is_conv and eval_precision == "f16":
            self._precision = "f16"
        if self._fused and not (self._is_conv or self._is_rnn or self._is_cnn or self._population) and \
                eval_precision != "fp32":
            probe = "eval_supports_f16" if eval_precision in ("auto", "f16") else "eval_supports_bf16"
            act_kw = {"act": self._act_code()} if self._act_code() else {}     # ReLU + MSE: the backends' default
            supported = getattr(self._be, probe, lambda d, b, **_: False)(self._spec.dims, self.agent.obs.shape[0],
                                                                          **act_kw)
            # "f16" where the cluster kernel's shape rule fails: the same arithmetic on the streamed kernel
            any_shape = (eval_precision == "f16" and not supported and
                         getattr(self._be, "eval_supports_f16_any", lambda d, b, **_: False)(
                             self._spec.dims, self.agent.obs.shape[0], **act_kw))
            if eval_precision != "auto" and not supported and not any_shape:
                raise ValueError(f"eval_precision={eval_precision!r} needs layer widths that are multiples of 64 "
                                 "(in) / 32 (out), at most 512 (f16: input width at most 256), and a batch that "
                                 "is a multiple of 256")
            self._precision = ("f16_any" if any_shape else
                               ("f16" if eval_precision == "auto" else eval_precision) if supported else "fp32")
            if eval_precision == "auto" and float(sigma) < AUTO_F16_MIN_SIGMA:
                self._precision = "fp32"

        # ---- noise table (replicated on every GPU, identical by construction)
        n_pad = (self.n_parameters + 31) // 32 * 32
        size = DEFAULT_NOISE_TABLE_SIZE if noise_table_size is None else int(noise_table_size)
        size = max(size, n_pad + 32) // 32 * 32
        self._table = self._be.alloc(size)
        self._be.fill_noise_table(self._table, self._noise_seed)
        self._table16 = None            # bf16 shadow ("bf16s" only)
        self._table16_version = None
        self._table_h = None            # EXACT fp16 copy of the table (None while unchecked / not exact)
        self._table_h_version, self._table_h_ok = None, False
        self._ensure_table16()

        # ---- population bookkeeping
        P, W = self.population_size, self.n_workers
        self._pairs = P // 2
        self._pairs_local = self._pairs // W
        self._pair_begin = self.rank * self._pairs_local
        be = self._be
        self._offsets = be.zeros(self._pairs_local, dtype=torch.int64)
        self._order = be.zeros(self._pairs_local, dtype=torch.int32)
        self._offsets_all = self._offsets if W == 1 else be.zeros(self._pairs, dtype=torch.int64)
        self._returns = be.zeros(P)
        self._novelty = None
        self._ranks = be.zeros(P, dtype=torch.int32)
        self._ranks2 = None
        self._grad = be.zeros(self.n_parameters)
        self._episode = be.zeros(1)
        self._obs = self._tgt = None
        if self._device_agent:
            self._obs = self.agent.obs.to(self._dev).contiguous()
            self._tgt = self.agent.target.to(self._dev).contiguous()
        self._data_obs = self._data_tgt = None
        if self._fused and self._sampling:
            # the whole dataset lives on the device; _obs / _tgt are the evaluate's batch buffers, refilled by
            # estk_sample_batch at the head of every generation
            self._data_obs = self.agent.dataset_obs.to(self._dev).contiguous()
            self._data_tgt = self.agent.dataset_target.to(self._dev).contiguous()

        self._xref = self._conv_scratch = self._conv_stats = None
        if self._fused and self._is_conv:
            self._xref = self.target.xref.detach().to(self._dev, torch.float32).contiguous()
        if self._fused and self._is_conv and self._population:
            # VBN statistics of every member, computed once per generation (population mode's conv act)
            self._conv_stats = torch.empty(P, ESTK_CONV_VBN_STATS_FLOATS, dtype=torch.float32, device=self._dev)
        elif self._fused and self._is_conv:
            nbytes = be.conv_scratch_bytes(self._xref.shape[0], self._obs.shape[0], self._precision)
            self._conv_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self._dev)

        self._slots = []
        if self._ALGORITHM_TYPE == _Algorithm.classic:
            self.policy = self._make_module()                       # estorch.py:136
            self.optimizer = optimizer(self.policy.parameters(), **optimizer_kwargs)   # :137
            self._slots.append(_PolicySlot(self.policy, self.optimizer, be, self._fused))
        self._active = self._slots[0] if self._slots else None
        self.step = 0
        self._generation = 0     # total generations ever run: indexes the noise offsets (never reset)
        self._pending_centre = False

    # ------------------------------------------------------------------ setup helpers
    def _make_module(self):
        module = self._policy_cls(**self._policy_kwargs)
        return module.to(self._dev if self._fused else self.device)

    def _hook_overridden(self, name):
        return not getattr(getattr(type(self), name), "_estk_builtin", False)

    def _decide_fused(self, optimizer_cls):
        """Fused mode for a DeviceAgent (an MLP, conv + VirtualBatchNorm or generic Conv2d + Linear policy) or a
        SequenceAgent (a recurrent policy), population mode for a PopulationAgent (a recognised MLP, conv +
        VirtualBatchNorm, recurrent or generic Conv2d + Linear policy on one GPU: the multi-GPU population
        generation is not implemented, hooks mode serves it).  A generic CNN is recognised for a DeviceAgent's
        images, and for a PopulationAgent that declares ``obs_shape``; a SequenceAgent with a CNN stays in hooks
        mode."""
        population = isinstance(self.agent, PopulationAgent)
        if not (self._device_agent or population) or self._spec is None:
            return False
        if population and self.n_workers > 1:
            return False
        # a recurrent policy is evaluated over sequences, other policies over a batch of observations
        if not population and self._is_rnn != isinstance(self.agent, SequenceAgent):
            return False
        if self._is_cnn and isinstance(self.agent, SequenceAgent):
            return False
        if optimizer_cls is not torch.optim.Adam:
            return False
        kw = self._optimizer_kwargs
        if any(kw.get(k) for k in _UNFUSED_ADAM_FLAGS):
            return False                        # the fused epilogue is Adam with L2 weight decay only
        if getattr(self, "k", 0) > 32:          # estk_knn_novelty's per-lane top-k buffer; the reference accepts
            return False                        # any k (estorch.py:413) -> hooks mode (host novelty) serves it
        if population:
            pass                                # its episodes are user code: no shape of the agent to check
        elif getattr(self.agent, "loss", "mse") in ("cross_entropy", "accuracy") and \
                (self._is_conv or self._spec.output != "identity"):
            return False                        # the logits are the output: identity-output MLPs and CNNs only
        elif self._is_conv:
            if self._ALGORITHM_TYPE != _Algorithm.classic:      # no behaviour characteristic on the conv kernel yet
                return False
            if tuple(self.agent.obs.shape[1:]) != (4, 84, 84) or \
                    tuple(self.agent.target.shape[1:]) != (self._spec.n_actions,):
                return False
        elif self._is_cnn:
            if tuple(self.agent.obs.shape[1:]) != self._spec.input_shape or \
                    tuple(self.agent.target.shape[1:]) != (self._spec.out,):
                return False
        elif self._is_rnn:
            if tuple(self.agent.obs.shape[2:]) != (self._spec.dims[0],) or \
                    tuple(self.agent.target.shape[2:]) != (self._spec.dims[-1],):
                return False
        elif tuple(self.agent.obs.shape[1:]) != (self._spec.dims[0],) or \
                tuple(self.agent.target.shape[1:]) != (self._spec.dims[-1],):
            return False
        hooks = ("_sample_policy", "_calculate_grad", "_calculate_returns", "_after_optimize",
                 "_get_policy", "_calculate_novelty", "_rollout_bc")
        return not any(hasattr(type(self), h) and self._hook_overridden(h) for h in hooks)

    # ------------------------------------------------------------------ reference API
    def terminate(self):
        """Stop training after the current generation (estorch.py:150-152)."""
        self._stop = True

    def log(self):
        """Called after every optimisation step; override to interact with
        training (estorch.py:154-172).  Reads below synchronise with the GPU."""
        print(f'Step: {self.step}')
        print(f'Episode Reward: {self.episode_reward}')
        print(f'Max Population Reward: {np.max(self.population_returns)}')
        print(f'Max Reward: {self.best_reward}')

    # -- lazily synchronised attributes (documented at estorch.py:108-117) --
    def _flush_pending_centre(self):
        """A deferred post-update rollout (see _fused_generation) is run now: something
        wants to observe episode_reward / the best snapshot before the next generation."""
        if getattr(self, "_pending_centre", False):
            slot = self._active
            self._eval_fns()[1](self._spec.dims, slot.theta, self._obs, self._tgt, self._episode,
                                **self._mlp_kw(slot, True))
            self._be.track_best(slot.state, self._episode, slot.theta, slot.best_theta)
            self._pending_centre = False
            self._host_cache = {}

    def _host_fetch(self):
        """Everything log() may read -- the population's returns (and novelty) and the active slot's
        ``estk_state`` -- in ONE device->host transfer per generation: asynchronous copies into pinned
        buffers, a single stream synchronisation, cached until the next generation."""
        self._flush_pending_centre()
        key = ("fetch", id(self._active), self.step, self._gen_token)
        if self._host_cache.get("key") == key:
            return self._host_cache
        rm = getattr(self, "_rm_live", False)      # multi-GPU fused runs keep the all-gathered (rank-major) layout
        cols = [self._returns_rm if rm else self._returns]
        if self._novelty is not None:
            cols.append(self._novelty_rm if rm else self._novelty)
        state = self._active.state if self._active is not None else None
        P = self.population_size
        if self._dev.type == "cuda":
            # raw device buffers -> pinned host memory, no staging kernel; re-ordering / stacking happen on the host
            pin = self.__dict__.setdefault("_pinned", {})
            if pin.get("shape") != (len(cols), P):
                pin.update(shape=(len(cols), P), ret=torch.empty(len(cols), P, dtype=torch.float32).pin_memory(),
                           state=torch.empty(32, dtype=torch.uint8).pin_memory())
            for i, c in enumerate(cols):
                pin["ret"][i].copy_(c.reshape(-1), non_blocking=True)
            if state is not None:
                pin["state"].copy_(state, non_blocking=True)
            torch.cuda.current_stream(self._dev).synchronize()
            raw = pin["ret"].numpy()
            st = read_state(pin["state"]) if state is not None else None
        else:
            raw = torch.stack([c.reshape(-1) for c in cols]).cpu().numpy()
            st = read_state(state) if state is not None else None
        if rm:      # [W][2][pairs/W] -> member order (all +, then all -: estorch.py:192)
            raw = raw.reshape(len(cols), self.n_workers, 2, self._pairs_local).transpose(0, 2, 1, 3).reshape(len(cols), P)
        host_ret = np.ascontiguousarray(raw.T)     # [P, 1] / [P, 2] like the reference's population_returns
        self._host_cache = {"key": key, "returns": host_ret, "state": st}
        return self._host_cache

    def _slot_state(self):
        return self._host_fetch()["state"]

    _gen_token = 0

    @property
    def episode_reward(self):
        if "_episode_reward" in self.__dict__:
            return self.__dict__["_episode_reward"]
        return self._slot_state()["episode_reward"]

    @episode_reward.setter
    def episode_reward(self, value):
        self.__dict__["_episode_reward"] = value

    @property
    def best_reward(self):
        if "_best_reward" in self.__dict__:
            return self.__dict__["_best_reward"]
        if self._fused and self._active is not None:
            return self._slot_state()["best_reward"]
        return -float("inf")

    @best_reward.setter
    def best_reward(self, value):
        self.__dict__["_best_reward"] = value

    @property
    def best_policy_dict(self):
        if "_best_policy_dict" in self.__dict__:
            return self.__dict__["_best_policy_dict"]
        self._flush_pending_centre()
        slot = self._best_slot if getattr(self, "_best_slot", None) is not None else self._active
        if slot is None or self.best_reward == -float("inf"):
            raise AttributeError("best_policy_dict is set after the first improving generation")
        out, idx = OrderedDict(), 0
        flat = slot.best_theta.detach().clone()
        names = [k for k, _ in slot.module.named_parameters()]
        sd = slot.module.state_dict()
        for k in sd:
            if k in names:
                sz = sd[k].numel()
                out[k] = flat[idx: idx + sz].view(sd[k].shape).clone()
                idx += sz
            else:
                out[k] = sd[k].detach().clone()
        return out

    @best_policy_dict.setter
    def best_policy_dict(self, value):
        self.__dict__["_best_policy_dict"] = value

    @property
    def population_returns(self):
        """np.float32 ``[P, 1]`` (ES) or ``[P, 2]`` = (reward, novelty) (NS family,
        estorch.py:441)."""
        if "_population_returns" in self.__dict__:
            return self.__dict__["_population_returns"]
        return self._host_fetch()["returns"]

    @population_returns.setter
    def population_returns(self, value):
        self.__dict__["_population_returns"] = value

    # ------------------------------------------------------------------ hooks (estorch.py:174-205)
    @_builtin
    def _get_policy(self):
        return self.policy, self.optimizer

    @_builtin
    def _sample_policy(self, policy):
        """-> (population_parameters, epsilon), both lazy ``[P, n]`` handles
        (estorch.py:187-193)."""
        slot = self._slot_of(policy)
        slot.push_theta()
        slot.theta_prev.copy_(slot.theta)
        self._draw_offsets()
        args = (self._be, slot.theta_prev, self._table, self._all_offsets(), self.sigma, self.population_size)
        return LazyPopulation(*args), NoiseHandle(*args)

    @_builtin
    def _calculate_returns(self, parameters):
        """Host rollouts over parameter rows (estorch.py:195-202)."""
        returns = []
        for parameter in parameters:
            torch.nn.utils.vector_to_parameters(parameter.to(self.device), self.target.parameters())
            returns.append(self.agent.rollout(self.target))
        return np.array(returns, dtype=np.float32)[:, np.newaxis]

    @_builtin
    def _calculate_grad(self, epsilon):
        """Flat gradient estimate ``(c @ eps) / (P*sigma)`` (estorch.py:174-179)."""
        return self._grad_from(epsilon, self.population_returns[:, 0], None, 1.0, 0.0)

    @_builtin
    def _after_optimize(self, policy):
        self.episode_reward = self.agent.rollout(policy)             # estorch.py:182
        if self.episode_reward > self.best_reward:
            self.best_reward = self.episode_reward
            self.best_policy_dict = copy.deepcopy(policy.state_dict())

    # ------------------------------------------------------------------ device helpers
    def _slot_of(self, policy):
        for s in self._slots:
            if s.module is policy:
                return s
        raise ValueError("policy is not managed by this ES instance")

    def _draw_offsets(self, state=None, gen_offset=0):
        """Offsets (and the offset-sorted order) of this generation's local pairs.  With
        ``state`` the generation index is read on the device (state.generation +
        gen_offset == self._generation), so the call can be replayed from a CUDA graph."""
        be = self._be
        self._offsets_gen = self._generation
        be.make_offsets(self._noise_seed, state, self._generation if state is None else gen_offset,
                        self._pair_begin, self._pairs_local,
                        self._table.numel(), self.n_parameters, self._offsets, self._order)
        self._offsets_all_gen = self._generation if self.n_workers == 1 else None

    def _all_offsets(self):
        """Offsets of ALL pairs of the last sampled population (lazy population rows);
        on multi-GPU runs they are only generated when somebody asks for rows."""
        if self.n_workers > 1 and getattr(self, "_offsets_all_gen", None) != self._offsets_gen:
            self._be.make_offsets(self._noise_seed, None, self._offsets_gen, 0, self._pairs,
                                  self._table.numel(), self.n_parameters, self._offsets_all, None)
            self._offsets_all_gen = self._offsets_gen
        return self._offsets_all

    def _grad_from(self, epsilon, rewards, novelty, w_rew, w_nov):
        """Gradient estimate for the hooks path: device reduction when ``epsilon``
        is the engine's NoiseHandle, dense matmul when a subclass supplied its
        own tensor."""
        P = self.population_size
        if not isinstance(epsilon, NoiseHandle):
            c = torch.from_numpy(rank_transformation(rewards)).float()
            if novelty is not None:
                c_nov = torch.from_numpy(rank_transformation(novelty)).float()
                c = w_rew * c + w_nov * c_nov
            eps = epsilon.to(torch.float32)
            return (torch.mm(c.unsqueeze(0).to(eps.device), eps) / (P * self.sigma)).squeeze()
        be = self._be
        self._returns.copy_(torch.as_tensor(np.ascontiguousarray(rewards, dtype=np.float32)))
        nov = None
        if novelty is not None:
            self._ensure_novelty()
            self._novelty.copy_(torch.as_tensor(np.ascontiguousarray(novelty, dtype=np.float32)))
            nov = self._novelty
        gsum = self._grad
        be.rank_grad(self._returns, nov, w_rew, w_nov, P, self._grad_table(), self._offsets, self._order,
                     self._pair_begin, self._pairs_local, self.n_parameters, gsum, self._ranks, self._ranks2)
        self._all_reduce(gsum)
        return gsum / float(P)

    def _ensure_novelty(self):
        if self._novelty is None:
            self._novelty = self._be.zeros(self.population_size)
            self._ranks2 = self._be.zeros(self.population_size, dtype=torch.int32)

    def _all_reduce(self, t):
        if self.n_workers > 1:
            import torch.distributed as dist
            dist.all_reduce(t)

    def _all_gather_halves(self, t):
        """Every rank wrote its local pairs' +/- members into ``t``; complete it with ONE
        all-gather (replaces the master's Recv loop, estorch.py:228-233)."""
        if self.n_workers == 1:
            return
        import torch.distributed as dist
        W, pl, pb, pairs = self.n_workers, self._pairs_local, self._pair_begin, self._pairs
        if getattr(self, "_gather_buf", None) is None or self._gather_buf.dtype != t.dtype:
            self._gather_buf = torch.empty(W, 2, pl, dtype=t.dtype, device=t.device)
            self._gather_loc = torch.empty(2, pl, dtype=t.dtype, device=t.device)
        loc = self._gather_loc
        loc[0].copy_(t[pb: pb + pl])
        loc[1].copy_(t[pairs + pb: pairs + pb + pl])
        dist.all_gather_into_tensor(self._gather_buf.view(-1), loc.view(-1))
        t.view(2, W, pl).copy_(self._gather_buf.permute(1, 0, 2))     # member order: all +, then all -

    def _sync_replicas(self):
        """Every rank constructs its own policy / meta-population (torch's default seed
        differs per process) while the reference keeps ONE master copy (estorch.py:136,
        :401-408): rank 0's state is authoritative and is broadcast before the loop, so
        that all ranks perturb the same centre and apply the same update."""
        if self.n_workers == 1:
            return
        # Fused mode keeps the replicas bit-identical by construction (same returns, same sum order, same Adam
        # bits on every rank), so a second train() call has nothing to broadcast: 20 MB + a pickled dict per
        # call was 3 % of a 20-generation run on 8 GPUs.  Hooks mode (host agents may be stochastic per rank)
        # and anything that rewrites the state (load_state_dict, sync_replicas()) synchronise again.
        if self._fused and getattr(self, "_replicas_synced", False):
            return
        import torch.distributed as dist
        for s_ in self._slots:
            s_.push_theta()
            for t in (s_.theta, s_.m, s_.v, s_.best_theta, s_.theta_prev, s_.state):
                dist.broadcast(t, src=0)
            if not s_.flattened:
                torch.nn.utils.vector_to_parameters(
                    s_.theta.detach().to(next(s_.module.parameters()).device).clone(), s_.module.parameters())
        host = {k: getattr(self, k) for k in ("_archive", "_best_host", "weight", "t", "_generation")
                if hasattr(self, k)}
        box = [host]
        dist.broadcast_object_list(box, src=0)
        for k, v in box[0].items():
            setattr(self, k, v)
        self._host_cache = {}
        self._replicas_synced = True

    def sync_replicas(self):
        """Make rank 0's parameters / optimizer state / algorithm state authoritative on every rank again (a
        collective: call it on every rank).  Needed only after rank 0's policy was modified by hand between two
        ``train()`` calls of a multi-GPU job; ``load_state_dict`` does it implicitly."""
        self._replicas_synced = False
        self._ensure_dist()
        for s_ in self._slots:
            s_.ensure_flat()
        self._sync_replicas()

    # -- rank-major returns: every rank's evaluate kernel writes its (+, -) halves straight into its
    #    block of a [W, 2, pairs/W] buffer, ONE in-place all-gather completes it, and the rank kernel
    #    (estk_rank_grad, `world`) reads that layout: no staging copies (estorch.py:228-233 Recv loop)
    def _member_order(self, t_rm):
        return t_rm.view(self.n_workers, 2, self._pairs_local).permute(1, 0, 2).reshape(-1)

    def _rm_buffers(self):
        if getattr(self, "_returns_rm", None) is None:
            self._returns_rm = self._be.zeros(self.n_workers, 2, self._pairs_local)
            self._novelty_rm = self._be.zeros(self.n_workers, 2, self._pairs_local) \
                if self._ALGORITHM_TYPE == _Algorithm.novelty else None
        return self._returns_rm, self._novelty_rm

    def _all_gather_rm(self, t_rm):
        import torch.distributed as dist
        dist.all_gather_into_tensor(t_rm.view(-1), t_rm[self.rank].reshape(-1))

    def _peer_workspaces(self):
        """Device pointers of every rank's cross-GPU workspace as mapped in this process (``estk.h``:
        estk_rank_grad_xr_adam sums the partial gradients over NVLink peer memory inside the kernel), or
        None when peer memory is not available -- then the NCCL all-reduce path runs.  Set up once, at the
        first fused generation, collectively: every rank takes the same decision."""
        if "_peer_ptrs" in self.__dict__:
            return self._peer_ptrs
        import torch.distributed as dist
        self._peer_ptrs = None
        be, W = self._be, self.n_workers
        mode = os.environ.get("ESTORCH_B200_PEER", "1")      # "0": NCCL; "force": also for small policies
        # (below ~1 MB of gradient the two cross-GPU barriers of the kernel cost as much as NCCL's small-message
        #  all-reduce: measured 51 vs 50 us at n = 214 k, 60 vs 45 us at n = 6 k, 212 vs 233 us at n = 1 M on 2 GPUs)
        ok = (self._dev.type == "cuda" and hasattr(be, "peer_alloc") and 2 <= W <= 16 and mode != "0"
              and (self.n_parameters >= (1 << 18) or mode == "force"))
        if not ok:            # decided by the job's configuration alone: the same on every rank, no collective
            return None
        mine = err = None
        if ok:
            try:
                mine = be.peer_alloc(be.xr_workspace_bytes(self.n_parameters))
            except Exception as e:      # no IPC in this container, out of memory, ...
                err = repr(e)
        handles = [None] * W
        dist.all_gather_object(handles, None if mine is None else mine[1])
        ptrs = None
        if all(h is not None for h in handles):
            try:
                ptrs = [mine[0] if r == self.rank else be.peer_open(handles[r]) for r in range(W)]
            except Exception as e:
                err = repr(e)
                ptrs = None
        flags = [None] * W
        dist.all_gather_object(flags, ptrs is not None)
        if all(flags):
            self._peer_ptrs = ptrs
        elif ok and self.rank == 0:
            import warnings
            warnings.warn(f"estorch_b200: NVLink peer memory unavailable ({err}); gradients are summed with NCCL")
        return self._peer_ptrs

    def _ensure_dist(self):
        if self.n_workers > 1:
            import torch.distributed as dist
            global _OWN_PROCESS_GROUP, _EXIT_HOOK
            _LIVE.add(self)
            if not dist.is_initialized():
                backend = "nccl" if self._dev.type == "cuda" else "gloo"
                dist.init_process_group(backend=backend)
                _OWN_PROCESS_GROUP = True
            if not _EXIT_HOOK:
                import atexit
                atexit.register(_shutdown_dist)
                _EXIT_HOOK = True

    def close(self):
        """Release what must go before ``torch.distributed.destroy_process_group()``: the CUDA graphs of the
        fused generation (they pin the NCCL communicator) and this process's mappings of the other ranks'
        peer-memory workspaces.  Call it on EVERY rank (it switches the gradient sum back to NCCL, which all
        ranks must agree on); training can continue afterwards (graphs are re-captured)."""
        self.__dict__.pop("_graphs", None)
        if self._dev.type == "cuda":
            torch.cuda.synchronize(self._dev)
        if hasattr(self._be, "peer_close_all") and self.__dict__.get("_peer_ptrs") is not None:
            self._be.peer_close_all()
            self._peer_ptrs = None

    # ------------------------------------------------------------------ fused generation
    def _adam_desc(self, optimizer):
        g = optimizer.param_groups[0]
        _refuse_unfused_adam_flags(g)
        return adam_desc(lr=g["lr"], betas=g["betas"], eps=g["eps"], weight_decay=g["weight_decay"], clamp=1.0)

    def _exact_table16(self):
        """The EXACT fp16 copy of the noise table, or None when some entry of the table is
        not fp16-representable (only tables written from outside: estk_fill_noise_table
        rounds every entry to fp16).  Consumers convert it back to fp32 exactly, so it is a
        drop-in for the fp32 table at half the bytes: the tensor-core evaluate streams it
        and so does the gradient reduction.  Re-checked when the table was overwritten in
        place (``tensor._version``); one host synchronisation per check (setup time)."""
        if self._table_h_version != self._table._version:
            if self._table_h is None:
                self._table_h = self._be.alloc(self._table.numel(), dtype=torch.float16)
            self._table_h_ok = self._be.shadow_f16(self._table, self._table_h) == 0
            self._table_h_version = self._table._version
        return self._table_h if self._table_h_ok else None

    def _grad_table(self):
        """Table the gradient reduction reads: the exact fp16 copy when there is one."""
        t = self._exact_table16() if hasattr(self._be, "shadow_f16") else None
        return self._table if t is None else t

    def _ensure_table16(self):
        """16-bit table copies of the tensor-core evaluate modes: ``"f16"`` / ``"f16_any"`` need the
        exact fp16 copy, ``"bf16s"`` a rounded bf16 shadow."""
        if self._precision in ("f16", "f16_any"):
            if self._exact_table16() is None:
                raise ValueError("eval_precision='f16' needs a noise table whose entries are exactly "
                                 "fp16-representable; use the engine's own table or eval_precision='fp32'")
        elif self._precision == "bf16s":
            if self._table16 is None or self._table16_version != self._table._version:
                if self._table16 is None:
                    self._table16 = self._be.alloc(self._table.numel(), dtype=torch.bfloat16)
                self._be.shadow_bf16(self._table, self._table16)
                self._table16_version = self._table._version

    def _eval_kw(self, slot, centre=False):
        """precision + the 16-bit table copy (and, for "bf16s", a refreshed bf16 shadow of
        theta) for the evaluate kernels."""
        kw = {"precision": self._precision}
        if self._precision == "bf16s":
            if slot.theta16 is None:
                slot.theta16 = self._be.alloc(slot.n, dtype=torch.bfloat16)
            self._be.shadow_bf16(slot.theta, slot.theta16)
            kw["theta16"] = slot.theta16
        if self._precision in ("f16", "f16_any", "bf16s") and not centre:
            self._ensure_table16()
            kw["table16"] = self._table16 if self._precision == "bf16s" else self._table_h
        return kw

    def _eval_fns(self):
        """(population, centre) evaluate of the fused generation: the recurrent sequence evaluate, the
        convolutional one or the MLP one (the same arguments)."""
        be = self._be
        if self._is_cnn:
            return be.eval_cnn, be.eval_cnn_center
        return (be.eval_rnn_seq, be.eval_rnn_seq_center) if self._is_rnn else (be.eval_mlp, be.eval_mlp_center)

    def _act_code(self):
        """``estk_mlp_desc.activation`` of the MLP evaluate: the policy's activations (include/estk.h
        ESTK_ACT_*) and the agent's loss (ESTK_LOSS_XENT for ``loss="cross_entropy"``, ESTK_LOSS_ACCURACY for
        ``loss="accuracy"``)."""
        loss = getattr(self.agent, "loss", "mse")
        return self._spec.act | {"cross_entropy": ESTK_LOSS_XENT, "accuracy": ESTK_LOSS_ACCURACY}.get(loss, 0)

    def _mlp_kw(self, slot, centre=False):
        """``_eval_kw`` plus the code of ``_act_code``.  It is left out for ReLU hidden + identity
        output + squared error, the default of every backend."""
        kw = self._eval_kw(slot, centre)
        if self._act_code():
            kw["act"] = self._act_code()
        return kw

    _streaming = False          # the agent hands a new observation batch to every generation
    _next_batch = None
    _next_batch_ptrs = None
    _peeked = False

    def _peek_batch(self):
        """Ask the agent for this generation's batch (host side, once per generation)."""
        if self._peeked:
            return
        self._peeked = True
        nb = self.agent.next_batch(self._generation)
        self._next_batch = nb
        self._streaming = nb is not None
        self._next_batch_ptrs = None if nb is None else (nb[0].data_ptr(), nb[1].data_ptr())
        if nb is not None:
            # a deferred post-update rollout belongs to the PREVIOUS batch (estorch.py:181-185
            # runs it before the next generation samples): run it before the buffers change
            self._flush_pending_centre()

    def _upload_batch(self):
        self._peek_batch()
        self._peeked = False
        nb, self._next_batch = self._next_batch, None
        if nb is not None:
            obs, tgt = nb
            self._obs.copy_(obs, non_blocking=True)
            self._tgt.copy_(tgt, non_blocking=True)

    def _update_step(self, slot, R, N, w_rew, w_nov, rm):
        """Ranks, gradient estimate and Adam step of a fused generation from the returns ``R`` (and the
        novelty ``N``, None for ES) -- rank-major ``[W, 2, pairs/W]`` buffers when ``rm``, member order
        otherwise.  One GPU: one launch.  Several: the rows are all-gathered, then ONE launch that also
        sums the gradient over NVLink peer memory, or, without peer memory, rank + partial gradient ->
        NCCL all-reduce -> clamp + Adam."""
        be, P, W, pb, pl = self._be, self.population_size, self.n_workers, self._pair_begin, self._pairs_local
        gt, ad = self._grad_table(), self._adam_desc(slot.optimizer)
        ranks2 = None if N is None else self._ranks2
        _nvtx_push("estk:rank_grad_adam")
        if W == 1:
            be.rank_grad_adam(R, N, w_rew, w_nov, P, gt, self._offsets, self._order,
                              slot.theta, slot.m, slot.v, slot.state, ad, self._ranks, ranks2, self._grad)
        else:
            peers = self._peer_workspaces() if rm else None
            gather = self._all_gather_rm if rm else self._all_gather_halves
            for t in ([R] if N is None else [R, N]):
                gather(t)
            nov = None if N is None else N.view(-1)
            if peers is not None:
                be.rank_grad_xr_adam(R.view(-1), nov, w_rew, w_nov, P, W, self.rank, gt, self._offsets, self._order,
                                     pb, pl, peers, slot.theta, slot.m, slot.v, slot.state, ad, self._ranks, ranks2,
                                     self._grad)
            else:
                be.rank_grad(R.view(-1), nov, w_rew, w_nov, P, gt, self._offsets, self._order, pb, pl,
                             self.n_parameters, self._grad, self._ranks, ranks2, world=W if rm else 1)
                self._all_reduce(self._grad)
                be.clamp_adam(self._grad, P, slot.theta, slot.m, slot.v, slot.state, ad, None)
        _nvtx_pop()

    def _defers_centre(self):
        """Whether this generation's post-update rollout (estorch.py:181-185) is deferred and folded into the
        next generation's evaluate launch: it is a single 30 us task, so it waits when nobody can observe it
        before then (no log() due, not the last generation, the observation batch does not change: never
        with minibatches, whose next batch is not this one).  Only the tensor-core MLP evaluate can carry it."""
        return (self._precision in ("f16", "bf16", "bf16s") and not self._is_conv and not self._stop
                and not self._streaming and not self._sampling
                and (self.step + 1) % self._log_interval != 0 and self.step + 1 < self.n_steps)

    def _fused_generation(self, slot):
        """One generation, entirely on the device (no host synchronisation).  The body only
        enqueues work whose arguments do not depend on host scalars that change from one
        generation to the next (the generation index and the Adam step live in
        ``estk_state``), so it can be captured once and replayed as a CUDA graph
        (``_graphed_generation``)."""
        be, pairs, pl, pb, W = self._be, self._pairs, self._pairs_local, self._pair_begin, self.n_workers
        dims = None if self._is_conv else self._spec.dims
        self._upload_batch()
        if self._sampling:    # this generation's minibatch: the generation index is read from slot.state
            be.sample_batch(self.agent.batch_seed, slot.state, 0, self._data_obs, self._obs, self._data_tgt,
                            self._tgt)
        slot.theta_prev.copy_(slot.theta)
        folded = self._pending_centre
        self._draw_offsets(slot.state, 1 if folded else 0)
        gt = self._grad_table()
        rm = W > 1 and gt.dtype == torch.float16
        self._rm_live = rm
        if rm:
            R = self._rm_buffers()[0]
            ret_p, ret_m = R[self.rank, 0], R[self.rank, 1]
        else:
            R = self._returns
            ret_p, ret_m = R[pb: pb + pl], R[pairs + pb: pairs + pb + pl]
        _nvtx_push("estk:evaluate")
        if self._is_conv:
            be.eval_conv_vbn(self._spec.n_actions, slot.theta, self._table, self._offsets, self._order, pl,
                             self.sigma, self._xref, self._obs, self._tgt, ret_p, ret_m, self._conv_scratch,
                             **self._eval_kw(slot))
        else:
            kw = self._mlp_kw(slot)
            if folded:        # the previous generation's post-update rollout rides in this launch
                kw["centre_out"] = self._episode
            self._eval_fns()[0](dims, slot.theta, self._table, self._offsets, self._order, pl, self.sigma,
                                self._obs, self._tgt, ret_p, ret_m, **kw)
            if folded:        # theta is still the previous update's result here (estorch.py:182-185)
                be.track_best(slot.state, self._episode, slot.theta, slot.best_theta)
                self._pending_centre = False
        _nvtx_pop()
        self._update_step(slot, R, None, 1.0, 0.0, rm)
        self._best_slot = slot
        if self._defers_centre():
            self._pending_centre = True
            return
        if self._is_conv:
            be.eval_conv_vbn(self._spec.n_actions, slot.theta, None, None, None, 1, 0.0, self._xref, self._obs,
                             self._tgt, self._episode, None, self._conv_scratch, **self._eval_kw(slot, True))
        else:
            self._eval_fns()[1](dims, slot.theta, self._obs, self._tgt, self._episode, **self._mlp_kw(slot, True))
        be.track_best(slot.state, self._episode, slot.theta, slot.best_theta)

    # ------------------------------------------------------------------ CUDA-graph replay of a generation
    def _graph_key(self, slot):
        """Everything a captured generation bakes in.  None = do not graph this generation."""
        if (not self._fused or self._dev.type != "cuda" or os.environ.get("ESTORCH_B200_GRAPH", "1") == "0"
                or getattr(self, "_graph_broken", False) or type(self)._fused_generation is not ES._fused_generation):
            return None
        g = slot.optimizer.param_groups[0]
        _refuse_unfused_adam_flags(g)           # a replay does not go through _adam_desc
        nb = self._next_batch_ptrs
        return (id(slot), bool(self._pending_centre), self._defers_centre(), float(g["lr"]), tuple(g["betas"]), float(g["eps"]),
                float(g["weight_decay"]), float(self.sigma), self._table._version, nb,
                self._obs.data_ptr(), self._tgt.data_ptr(), torch.cuda.current_stream(self._dev).cuda_stream)

    def _graphed_generation(self, slot):
        """Run one fused generation: eagerly the first two times a configuration is seen, then
        captured into a CUDA graph and replayed (one launch instead of ~10 + 2 collectives;
        at 8 GPUs the host-side launch cost was 40 % of a generation)."""
        if self._population:        # the episode loop is host code: nothing to capture
            return self._population_generation(slot)
        self._peek_batch()
        key = self._graph_key(slot)
        if key is None:
            return self._fused_generation(slot)
        cache = self.__dict__.setdefault("_graphs", {})
        ent = cache.get(key)
        if not isinstance(ent, tuple):
            # A configuration is captured at its THIRD sighting: the first two run eagerly (they warm every lazy
            # allocation, and the configurations that occur once per train() call -- first / last generation --
            # never pay for a capture, which costs tens of milliseconds)
            if ent is None and len(cache) >= 8:    # configurations keep changing (e.g. an lr schedule): stay eager
                return self._fused_generation(slot)
            cache[key] = (ent or 0) + 1
            if cache[key] < 3:
                return self._fused_generation(slot)
            try:
                graph = torch.cuda.CUDAGraph()
                launches0 = self._be.launches
                pending0 = self._pending_centre
                cur, side = torch.cuda.current_stream(self._dev), self._graph_stream()
                side.wait_stream(cur)
                with torch.cuda.stream(side):   # (capture_begin/end directly: torch.cuda.graph() would also run
                    graph.capture_begin()       #  gc.collect() + empty_cache() + a device synchronize)
                    try:
                        self._fused_generation(slot)
                    finally:
                        graph.capture_end()
                cur.wait_stream(side)
                ent = cache[key] = (graph, self._be.launches - launches0, self._pending_centre, self._rm_live)
                self._pending_centre = pending0
                self._be.launches = launches0
            except Exception as e:            # capture is an optimisation: never a reason to stop training
                self._graph_broken = True
                cache.pop(key, None)
                import warnings
                warnings.warn(f"estorch_b200: CUDA-graph capture of a generation failed ({e!r}); running eagerly")
                torch.cuda.synchronize(self._dev)
                return self._fused_generation(slot)
        graph, n_launches, pending_after, rm_live = ent
        graph.replay()
        self._be.launches += n_launches
        self._pending_centre = pending_after
        self._rm_live = rm_live
        self._offsets_gen = self._generation
        self._offsets_all_gen = self._generation if self.n_workers == 1 else None
        self._best_slot = slot

    # ------------------------------------------------------------------ population generation (PopulationAgent)
    def _population_act(self, slot, centre=False):
        """The ``act`` handed to ``rollout_population``: observations ``[M, in]`` or ``[M, B, in]`` -> outputs of
        every member in ONE launch (estk_eval_mlp with ESTK_ACTIONS).  Population: M = P members of the last
        drawn offsets around ``slot.theta_prev`` (+ members first, then their mirrors); centre: M = 1, theta."""
        if self._is_conv:
            return self._population_act_conv(slot, centre)
        if self._is_rnn:
            return self._population_act_rnn(slot, centre)
        if self._is_cnn:
            return self._population_act_cnn(slot, centre)
        be, dims, dev, code = self._be, self._spec.dims, self._dev, self._spec.act
        M = 1 if centre else self.population_size
        t16 = None if centre or not hasattr(be, "shadow_f16") else self._exact_table16()

        def act(obs):
            x = torch.as_tensor(obs).to(device=dev, dtype=torch.float32).contiguous()
            single = x.dim() == 2
            x3 = x.unsqueeze(1) if single else x
            if x3.dim() != 3 or x3.shape[0] != M or x3.shape[2] != dims[0]:
                raise ValueError(f"act: observations {tuple(x.shape)}, expected [{M}, {dims[0]}] or "
                                 f"[{M}, B, {dims[0]}]")
            out = torch.empty(M, x3.shape[1], dims[-1], dtype=torch.float32, device=dev)
            if centre:
                be.act_mlp(dims, slot.theta, None, None, None, 1, 0.0, x3, out, act=code)
            else:
                be.act_mlp(dims, slot.theta_prev, self._table, self._offsets, self._order, self._pairs_local,
                           self.sigma, x3, out, act=code, table16=t16)
            return out[:, 0] if single else out
        return act

    def _population_act_rnn(self, slot, centre):
        """``act(obs, state=None) -> (out, new_state)`` for a recurrent policy (RNNSpec): observations ``[M, in]``
        or ``[M, B, in]``, the state h (GRU) or (h, c) (LSTM) of ``[M, H]`` or ``[M, B, H]`` tensors, None for
        zeros.  One launch per call: the kernel's rows are [x | state] -> [y | state'] (estk_eval_mlp with
        ESTK_CELL_GRU / ESTK_CELL_LSTM and ESTK_ACTIONS); the returned outputs and state are views of its
        output rows."""
        be, dev, spec = self._be, self._dev, self._spec
        (din, H, dout), lstm = spec.dims, spec.cell == "lstm"
        M = 1 if centre else self.population_size
        # the fp32 table, not its fp16 copy: the step forms its tiles from scalar noise loads and is not bound by
        # their bytes, and with the fp16 copy the LSTM step measured slower (DESIGN §9)

        def act(obs, state=None):
            x = torch.as_tensor(obs).to(device=dev, dtype=torch.float32)
            single = x.dim() == 2
            x3 = x.unsqueeze(1) if single else x
            if x3.dim() != 3 or x3.shape[0] != M or x3.shape[2] != din:
                raise ValueError(f"act: observations {tuple(x.shape)}, expected [{M}, {din}] or [{M}, B, {din}]")
            lead = tuple(x.shape[:-1])
            if state is None:
                parts = [torch.zeros(*lead, H * (2 if lstm else 1), dtype=torch.float32, device=dev)]
            else:
                parts = list(state) if lstm else [state]
                if len(parts) != (2 if lstm else 1) or any(not torch.is_tensor(p_) or tuple(p_.shape) != lead + (H,)
                                                           for p_ in parts):
                    want = f"(h, c), each [{', '.join(map(str, lead + (H,)))}]" if lstm else \
                        f"h [{', '.join(map(str, lead + (H,)))}]"
                    raise ValueError(f"act: the state must be None or {want}")
                parts = [p_.to(device=dev, dtype=torch.float32) for p_ in parts]
            xs = torch.cat([x] + parts, -1)
            xs = (xs.unsqueeze(1) if single else xs).contiguous()
            out = torch.empty(M, xs.shape[1], dout + spec.state_width, dtype=torch.float32, device=dev)
            if centre:
                be.act_rnn(spec.dims, slot.theta, None, None, None, 1, 0.0, xs, out, spec.act)
            else:
                be.act_rnn(spec.dims, slot.theta_prev, self._table, self._offsets, self._order, self._pairs_local,
                           self.sigma, xs, out, spec.act)
            if single:
                out = out[:, 0]
            y, h = out[..., :dout], out[..., dout:dout + H]
            return y, ((h, out[..., dout + H:]) if lstm else h)
        return act

    def _population_act_cnn(self, slot, centre):
        """``act`` for a Conv2d stack + Linear head policy (CNNSpec): images ``[M, c, h, w]`` or
        ``[M, B, c, h, w]`` -> outputs ``[M, out]`` or ``[M, B, out]``, one estk_act_cnn launch per call."""
        be, dev, spec = self._be, self._dev, self._spec
        M = 1 if centre else self.population_size
        shape = tuple(spec.input_shape)

        def act(obs):
            x = torch.as_tensor(obs).to(device=dev, dtype=torch.float32).contiguous()
            single = x.dim() == 4
            x5 = x.unsqueeze(1) if single else x
            if x5.dim() != 5 or x5.shape[0] != M or tuple(x5.shape[2:]) != shape:
                dims = ", ".join(map(str, shape))
                raise ValueError(f"act: images {tuple(x.shape)}, expected [{M}, {dims}] or [{M}, B, {dims}]")
            out = torch.empty(M, x5.shape[1], spec.out, dtype=torch.float32, device=dev)
            if centre:
                be.act_cnn(spec.dims, slot.theta, None, None, None, 1, 0.0, x5, out, spec.act)
            else:
                be.act_cnn(spec.dims, slot.theta_prev, self._table, self._offsets, self._order, self._pairs_local,
                           self.sigma, x5, out, spec.act)
            return out[:, 0] if single else out
        return act

    def _population_act_conv(self, slot, centre):
        """``act`` for the conv + VirtualBatchNorm policy: frames ``[M, 4, 84, 84]`` or ``[M, B, 4, 84, 84]`` ->
        outputs ``[M, A]`` or ``[M, B, A]``.  The members' VBN statistics over ``xref`` depend only on their
        weights, so they are computed by ONE launch here, when the ``act`` is built, and every call is one
        launch that reuses them (the reference recomputes them on every forward, examples/atari.py:25-37).
        The centre form keeps them in a one-member buffer of its slot."""
        be, dev, A = self._be, self._dev, self._spec.n_actions
        M = 1 if centre else self.population_size
        t16 = None if centre or not hasattr(be, "shadow_f16") else self._exact_table16()
        if centre:
            if getattr(slot, "conv_stats", None) is None:
                slot.conv_stats = torch.empty(1, ESTK_CONV_VBN_STATS_FLOATS, dtype=torch.float32, device=dev)
            theta, stats, args = slot.theta, slot.conv_stats, (None, None, None, 1, 0.0)
        else:
            theta, stats = slot.theta_prev, self._conv_stats
            args = (self._table, self._offsets, self._order, self._pairs_local, self.sigma)
        be.act_conv_vbn(A, theta, *args, self._xref, None, None, stats, table16=t16)

        def act(obs):
            x = torch.as_tensor(obs).to(device=dev, dtype=torch.float32).contiguous()
            single = x.dim() == 4
            x5 = x.unsqueeze(1) if single else x
            if x5.dim() != 5 or x5.shape[0] != M or tuple(x5.shape[2:]) != (4, 84, 84):
                raise ValueError(f"act: frames {tuple(x.shape)}, expected [{M}, 4, 84, 84] or [{M}, B, 4, 84, 84]")
            out = torch.empty(M, x5.shape[1], A, dtype=torch.float32, device=dev)
            be.act_conv_vbn(A, theta, *args, None, x5, out, stats, table16=t16)
            return out[:, 0] if single else out
        return act

    def _population_rollout(self, slot, centre=False):
        """``rollout_population`` of the agent -> (returns ``[M]``, bc ``[M, bc_dim]`` or None) on the device."""
        M = 1 if centre else self.population_size
        res = self.agent.rollout_population(self._population_act(slot, centre), M)
        ret, bc = res if self._ALGORITHM_TYPE == _Algorithm.novelty else (res, None)
        ret = torch.as_tensor(ret).to(device=self._dev, dtype=torch.float32).reshape(M)
        if bc is not None:
            bc = torch.as_tensor(bc).to(device=self._dev, dtype=torch.float32).reshape(M, -1)
        return ret, bc

    def _population_centre(self, slot):
        """theta's rollout into ``self._episode`` (NS family: and its behaviour characteristic into
        ``self._bc_center[0]``) -- what eval_mlp_center writes in fused mode."""
        ret, bc = self._population_rollout(slot, centre=True)
        self._episode.copy_(ret)
        if bc is not None:
            self._bc_center.copy_(bc)

    def _population_generation(self, slot):
        """One generation with a PopulationAgent (one GPU): offsets, the agent's episodes of all P members
        (every step one fused launch), returns (and novelty) into the member-order buffers, the fused
        rank + gradient + Adam step, then theta's rollout and the best tracking."""
        be, pl = self._be, self._pairs_local
        slot.theta_prev.copy_(slot.theta)
        self._draw_offsets()
        self._rm_live = False
        ret, bc = self._population_rollout(slot)
        self._returns.copy_(ret)
        novelty = self._ALGORITHM_TYPE == _Algorithm.novelty
        if novelty:
            self._bc.copy_(bc)
            be.knn_novelty(self._bc[:pl], self._arch_dev, self.k, self._novelty[:pl])
            be.knn_novelty(self._bc[pl:], self._arch_dev, self.k, self._novelty[pl:])
            self._update_step(slot, self._returns, self._novelty, np.float32(self._w_rew()),
                              np.float32(self._w_nov()), False)
            self._population_centre(slot)
            self._after_update(slot)
            return
        self._update_step(slot, self._returns, None, 1.0, 0.0, False)
        self._best_slot = slot
        self._population_centre(slot)
        be.track_best(slot.state, self._episode, slot.theta, slot.best_theta)

    def _graph_stream(self):
        if getattr(self, "_gstream", None) is None:
            self._gstream = torch.cuda.Stream(self._dev)
        return self._gstream

    @property
    def population_parameters(self):
        """Lazy ``[P, n]`` view of the last sampled population (estorch.py:216)."""
        if "_population_parameters" in self.__dict__:
            return self.__dict__["_population_parameters"]
        slot = self._active
        return LazyPopulation(self._be, slot.theta_prev, self._table, self._all_offsets(), self.sigma,
                              self.population_size)

    @population_parameters.setter
    def population_parameters(self, value):
        self.__dict__["_population_parameters"] = value

    # ------------------------------------------------------------------ hooks-mode generation
    def _hooks_generation(self):
        """The reference's control flow (estorch.py:215-246) through its hooks."""
        policy, optimizer = self._get_policy()
        if self.n_workers > 1 and self._ALGORITHM_TYPE == _Algorithm.novelty:
            # only the reference's master selects the meta-policy (estorch.py:444-456)
            import torch.distributed as dist
            box = [getattr(self, "idx", 0)]
            dist.broadcast_object_list(box, src=0)
            self.idx = int(box[0])
            self._active = self._slots[self.idx]
            policy, optimizer = self.meta_population[self.idx]
        self.population_parameters, epsilon = self._sample_policy(policy)
        per = self.population_size // self.n_workers
        pop = self.population_parameters
        if isinstance(pop, LazyPopulation):
            # a rank owns pairs, i.e. the matching +/- rows (estorch.py:217-223 sends
            # contiguous row blocks instead; the set of evaluated members is the same)
            pl, pb, pairs = self._pairs_local, self._pair_begin, self._pairs
            plus = self._calculate_returns(pop.rows(pb, pl))
            minus = self._calculate_returns(pop.rows(pairs + pb, pl))
            width = plus.shape[1]
            full = np.empty((self.population_size, width), dtype=np.float32)
            full[pb: pb + pl], full[pairs + pb: pairs + pb + pl] = plus, minus
            if self.n_workers > 1:
                t = torch.from_numpy(full).to(self._dev)
                for c in range(width):
                    col = t[:, c].contiguous()
                    self._all_gather_halves(col)
                    t[:, c] = col
                full = t.cpu().numpy()
            self.population_returns = full
        else:
            start = self.rank * per
            returns = self._calculate_returns(pop[start: start + per])
            if self.n_workers > 1:
                import torch.distributed as dist
                parts = [None] * self.n_workers
                dist.all_gather_object(parts, returns)
                returns = np.concatenate(parts)
            self.population_returns = returns
        grad = self._calculate_grad(epsilon)
        index = 0
        for parameter in policy.parameters():                         # estorch.py:236-244
            size = int(np.prod(parameter.shape))
            parameter.grad = (-grad[index:index + size].view(parameter.shape).to(parameter.device))
            parameter.grad.data.clamp_(-1.0, 1.0)
            index += size
        optimizer.step()                                              # estorch.py:245
        self._after_optimize(policy)
        if self.n_workers > 1 and self._ALGORITHM_TYPE == _Algorithm.novelty:
            # the master's post-update rollout is the one that enters the archive and drives
            # the NSRA schedule (estorch.py:427-432, :458-471 broadcast the archive)
            import torch.distributed as dist
            box = [{k: getattr(self, k) for k in ("episode_reward", "best_reward", "weight", "t") if hasattr(self, k)}
                   | {"bc": self._archive[-1]}]
            dist.broadcast_object_list(box, src=0)
            self._archive[-1] = box[0].pop("bc")
            for k, v in box[0].items():
                setattr(self, k, v)

    # ------------------------------------------------------------------ main loop
    def _master(self):
        """Generation loop (estorch.py:211-250).  Every rank runs it; only rank 0
        calls ``log`` (the reference's workers have no log either)."""
        self.step = 0
        self._ensure_dist()
        for s in self._slots:
            s.ensure_flat()
        self._sync_replicas()
        with torch.no_grad():
            while self.step < self.n_steps and not self._stop:
                self._gen_token += 1
                if self._fused:
                    for k in ("_episode_reward", "_best_reward", "_best_policy_dict",
                              "_population_returns", "_population_parameters"):
                        self.__dict__.pop(k, None)
                    self._active = self._select_slot()
                    self._graphed_generation(self._active)
                else:
                    if self._sampling:      # host rollouts see the minibatch the fused generation would gather
                        self.agent.set_generation(self._generation)
                    self._hooks_generation()
                if (self.step + 1) % self._log_interval == 0:
                    if self.rank == 0:
                        self.log()
                    self._sync_stop()
                self.step += 1
                self._generation += 1
        if self._fused:
            for s in self._slots:
                s.mirror_adam_state()
            torch.cuda.synchronize(self._dev) if self._dev.type == "cuda" else None

    def _select_slot(self):
        return self._slots[0]

    def _stop_channel(self):
        """A 16-byte shared-memory segment (all ranks of a torchrun job live on one host): rank 0 publishes
        (sequence number, stop flag) after ``log()``, the others read it -- no collective, no GPU round trip in
        the per-generation path.  None when a rank cannot map it (then ``_sync_stop`` broadcasts)."""
        if "_stop_shm" in self.__dict__:
            return self._stop_shm
        import torch.distributed as dist
        from multiprocessing import shared_memory
        self._stop_shm = None
        name, shm = [None], None
        if os.environ.get("ESTORCH_B200_STOP_SHM", "1") != "0":
            try:
                if self.rank == 0:
                    shm = shared_memory.SharedMemory(create=True, size=16)
                    shm.buf[:16] = bytes(16)
                    name = [shm.name]
            except Exception:
                name = [None]
        dist.broadcast_object_list(name, src=0)
        if self.rank != 0 and name[0] is not None:
            try:
                shm = shared_memory.SharedMemory(name=name[0])
                try:        # the creator unlinks it; attaching must not register a second owner (bpo-39959)
                    from multiprocessing import resource_tracker
                    resource_tracker.unregister(shm._name, "shared_memory")
                except Exception:
                    pass
            except Exception:
                shm = None
        oks = [None] * self.n_workers
        dist.all_gather_object(oks, shm is not None)
        if all(oks):
            self._stop_shm = (shm, np.ndarray((2,), dtype=np.int64, buffer=shm.buf), [0])
            import atexit
            atexit.register(_release_shm, shm, self.rank == 0)
        elif shm is not None:
            _release_shm(shm, self.rank == 0)
        return self._stop_shm

    def _sync_stop(self):
        """Rank 0's ``terminate()`` must stop every rank at the same generation."""
        if self.n_workers > 1:
            import torch.distributed as dist
            ch = self._stop_channel()
            if ch is not None:
                _, words, seq = ch
                seq[0] += 1
                if self.rank == 0:
                    words[1] = 1 if self._stop else 0      # flag first, sequence number second (x86 keeps the order)
                    words[0] = seq[0]
                else:
                    t0 = time.monotonic()
                    while words[0] < seq[0]:
                        if time.monotonic() - t0 > 600.0:
                            raise RuntimeError("estorch_b200: rank 0 did not publish its stop flag within 600 s")
                    self._stop = bool(words[1])
                return
            if self._dev.type != "cuda":
                flag = torch.tensor([1.0 if self._stop else 0.0])
                dist.broadcast(flag, src=0)
                self._stop = bool(flag.item() > 0)
                return
            # pinned host word -> device word -> broadcast -> pinned host word: no allocation, one synchronisation
            sf = self.__dict__.get("_stop_bufs")
            if sf is None:
                sf = self._stop_bufs = (torch.zeros(1).pin_memory(), torch.zeros(1, device=self._dev),
                                        torch.zeros(1).pin_memory())
            src, dev, dst = sf
            if self.rank == 0:
                src[0] = 1.0 if self._stop else 0.0
                dev.copy_(src, non_blocking=True)
            dist.broadcast(dev, src=0)
            dst.copy_(dev, non_blocking=True)
            torch.cuda.current_stream(self._dev).synchronize()
            self._stop = bool(dst[0] > 0)

    def train(self, n_steps, n_proc=1, hwthread=False, hostfile=None):
        """Train for ``n_steps`` generations (estorch.py:272-308).

        ``n_proc`` is the number of GPUs (one process per GPU).  Like the
        reference, which re-executes the calling script under ``mpirun``
        (estorch.py:41-56,:305), a single-process call with ``n_proc > 1``
        re-executes the script under ``torch.distributed.run`` and exits; when
        already running under a launcher (``WORLD_SIZE`` set) it just trains.
        ``hwthread`` is accepted and ignored; ``hostfile`` (multi-node MPI) is
        not supported.
        """
        self.n_steps = n_steps
        if hostfile is not None:
            raise NotImplementedError("hostfile (multi-node MPI launch) has no single-box equivalent here")
        if n_proc > 1:
            if self._trained:
                raise RuntimeError("train function can not be called more than once.")
            self._trained = True
            if self.n_workers == 1:
                from .launch import fork_under_torchrun
                if fork_under_torchrun(n_proc):
                    sys.exit(0)
            elif self.n_workers != n_proc:
                raise RuntimeError(f"train(n_proc={n_proc}) but the launcher started {self.n_workers} processes")
        self._master()


    # ------------------------------------------------------------------ checkpoint / resume
    # (the reference keeps everything in memory only, SURVEY 5; users pickle from log())
    def state_dict(self):
        """Everything needed to continue training bit-identically: theta / Adam moments /
        step counters / best snapshot per (policy, optimizer) slot, the generation
        counter and noise seed (the table is regenerated from the seed), and the host
        scalars of the algorithm."""
        self._flush_pending_centre()
        self._host_cache = {}
        slots = []
        for s_ in self._slots:
            s_.push_theta()
            st = read_state(s_.state)
            slots.append({"theta": s_.theta.detach().cpu().clone(), "m": s_.m.detach().cpu().clone(),
                          "v": s_.v.detach().cpu().clone(), "best_theta": s_.best_theta.detach().cpu().clone(),
                          "state": st,
                          "optimizer": None if s_.flattened else copy.deepcopy(s_.optimizer.state_dict())})
        out = {"version": 1, "algorithm": type(self).__name__, "n_parameters": self.n_parameters,
               "population_size": self.population_size, "sigma": self.sigma, "noise_seed": self._noise_seed,
               "noise_table_size": self._table.numel(), "generation": self._generation, "slots": slots,
               "best_reward": self.best_reward, "numpy_rng": np.random.get_state()}
        for k in ("_archive", "idx", "weight", "t", "_best_host"):
            if hasattr(self, k):
                out[k] = copy.deepcopy(getattr(self, k))
        if "_best_policy_dict" in self.__dict__:
            out["best_policy_dict"] = {k: v.detach().cpu().clone() for k, v in self.__dict__["_best_policy_dict"].items()}
        return out

    def load_state_dict(self, sd):
        if sd.get("algorithm") != type(self).__name__ or sd["n_parameters"] != self.n_parameters or \
                sd["population_size"] != self.population_size or len(sd["slots"]) != len(self._slots):
            raise ValueError("checkpoint does not match this algorithm / policy / population")
        if sd["noise_seed"] != self._noise_seed or sd["noise_table_size"] != self._table.numel():
            raise ValueError("checkpoint was written with a different noise table (seed or size)")
        self.sigma = sd["sigma"]
        self._replicas_synced = False
        self._generation = int(sd["generation"])
        for s_, rec in zip(self._slots, sd["slots"]):
            s_.ensure_flat()
            s_.theta.copy_(rec["theta"]); s_.m.copy_(rec["m"]); s_.v.copy_(rec["v"])
            s_.best_theta.copy_(rec["best_theta"])
            write_state(s_.state, **rec["state"])
            if not s_.flattened:
                torch.nn.utils.vector_to_parameters(rec["theta"].to(next(s_.module.parameters()).device).clone(),
                                                    s_.module.parameters())
                if rec["optimizer"] is not None:
                    s_.optimizer.load_state_dict(rec["optimizer"])
            else:
                s_.mirror_adam_state()
        for k in ("_archive", "idx", "weight", "t", "_best_host"):
            if k in sd:
                setattr(self, k, copy.deepcopy(sd[k]))
        if not self._fused or self._ALGORITHM_TYPE == _Algorithm.novelty:
            self.best_reward = sd["best_reward"]
        if "best_policy_dict" in sd:
            self.best_policy_dict = {k: v.clone() for k, v in sd["best_policy_dict"].items()}
        np.random.set_state(sd["numpy_rng"])
        self._host_cache = {}

    def save_checkpoint(self, path):
        if self.rank == 0:
            torch.save(self.state_dict(), path)

    def load_checkpoint(self, path):
        self.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))


class NS_ES(ES):
    """Novelty Search ES (Conti et al. 2018) -- reference estorch.py:311-472.
    Maintains a meta-population of ``meta_population_size`` (policy, optimizer)
    pairs and an archive of behaviour characteristics; the gradient follows
    novelty only.  ``population_returns`` is ``[P, 2]`` = (reward, novelty)."""

    _ALGORITHM_TYPE = _Algorithm.novelty
    _W_REW, _W_NOV = 0.0, 1.0

    def __init__(self, policy, agent, optimizer, population_size, sigma=0.01,
                 meta_population_size=3, k=10, device=torch.device("cpu"),
                 policy_kwargs={}, agent_kwargs={}, optimizer_kwargs={}, **engine_kwargs):
        self.meta_population_size = meta_population_size
        self.k = k            # known before _decide_fused(): the device kNN keeps k <= 32 neighbours
        super().__init__(policy, agent, optimizer, population_size, sigma, device,
                         policy_kwargs, agent_kwargs, optimizer_kwargs, **engine_kwargs)
        self._archive = []
        self.meta_population = []
        self._ensure_novelty()
        if self._fused:
            bc_dim = self.agent.bc_dim
            if not bc_dim:
                raise ValueError("NS-family device agents need bc_obs / bc_dim")
            self._bc = self._be.zeros(self.population_size, bc_dim)
            self._bc_center = self._be.zeros(1, bc_dim)
            self._nov_center = self._be.zeros(1)
        for _ in range(self.meta_population_size):                    # estorch.py:401-408
            p = self._make_module()
            optim = optimizer(p.parameters(), **optimizer_kwargs)
            self.meta_population.append((p, optim))
            self._slots.append(_PolicySlot(p, optim, self._be, self._fused))
            reward, bc = self._rollout_bc(p)
            if bc is None:
                raise ValueError("Behaviour Charateristics is None")
            self._archive.append(bc)
        self._active = self._slots[0]
        self._best_host = -float("inf")

    @_builtin
    def _rollout_bc(self, policy):
        """Initial archive entry of a meta-population member (estorch.py:405)."""
        if self._fused:
            self._centre_bc(self._slots[-1])
            return float(self._episode.item()), self._bc_center[0].cpu().numpy().copy()
        with torch.no_grad():
            return self.agent.rollout(policy)

    # -- host novelty (estorch.py:412-417), brute force in float64
    @_builtin
    def _calculate_novelty(self, bc, _archive):
        a = np.asarray(_archive, dtype=np.float64)
        d = np.sqrt(((a - np.asarray(bc, dtype=np.float64)[None, :]) ** 2).sum(axis=1))
        d.sort()
        return np.sum(d[:self.k]) / np.linalg.norm(a)

    @_builtin
    def _calculate_grad(self, epsilon):
        r = self.population_returns
        return self._grad_from(epsilon, r[:, 0], r[:, 1], np.float32(self._w_rew()), np.float32(self._w_nov()))

    def _w_rew(self):
        return self._W_REW

    def _w_nov(self):
        return self._W_NOV

    @_builtin
    def _after_optimize(self, policy):
        self.episode_reward, bc = self.agent.rollout(policy)          # estorch.py:427-432
        self._archive.append(bc)
        if self.episode_reward > self.best_reward:
            self.best_reward = self.episode_reward
            self.best_policy_dict = copy.deepcopy(policy.state_dict())

    @_builtin
    def _calculate_returns(self, parameters):
        returns = []
        for parameter in parameters:                                  # estorch.py:434-442
            torch.nn.utils.vector_to_parameters(parameter.to(self.device), self.target.parameters())
            reward, bc = self.agent.rollout(self.target)
            returns.append((reward, self._calculate_novelty(bc, self._archive)))
        return np.array(returns, dtype=np.float32)

    @_builtin
    def _get_policy(self):
        total_novelty = []                                            # estorch.py:444-456
        for policy, _ in self.meta_population:
            reward, bc = self.agent.rollout(policy)
            total_novelty.append(self._calculate_novelty(bc, self._archive))
        total_novelty = np.array(total_novelty)
        probability = total_novelty / np.sum(total_novelty)
        self.idx = np.random.choice(np.arange(len(self.meta_population), dtype=int), p=probability)
        self._active = self._slots[self.idx]
        return self.meta_population[self.idx]

    # ------------------------------------------------------------------ fused NS generation
    def _centre_bc(self, slot):
        """Rollout of ``slot``'s theta: its return into ``self._episode``, its behaviour characteristic into
        ``self._bc_center[0]`` (the device kernel in fused mode, the agent's episodes in population mode)."""
        if self._population:
            return self._population_centre(slot)
        ag = self.agent
        self._eval_fns()[1](self._spec.dims, slot.theta, self._obs, self._tgt, self._episode,
                            self._bc_center[0], ag.bc_obs, ag.bc_dim, **self._mlp_kw(slot, True))

    def _archive_tensor(self):
        return torch.from_numpy(np.ascontiguousarray(np.stack(self._archive), dtype=np.float32)).to(self._dev)

    def _select_slot(self):
        """Device version of ``_get_policy``: M centre rollouts + kNN novelty,
        then the reference's ``np.random.choice`` on the host (estorch.py:451-454)."""
        be = self._be
        arch = self._archive_tensor()
        nov = []
        for s in self._slots:
            self._centre_bc(s)
            be.knn_novelty(self._bc_center, arch, self.k, self._nov_center)
            nov.append(self._nov_center.clone())
        total = torch.cat(nov).double().cpu().numpy()
        self.idx = np.random.choice(np.arange(len(self.meta_population), dtype=int), p=total / np.sum(total))
        if self.n_workers > 1:                      # every rank must pick the same policy
            import torch.distributed as dist
            t = torch.tensor([self.idx], device=self._dev)
            dist.broadcast(t, src=0)
            self.idx = int(t.item())
        self._arch_dev = arch
        return self._slots[self.idx]

    def _fused_generation(self, slot):
        be, pairs, pl, pb, W = self._be, self._pairs, self._pairs_local, self._pair_begin, self.n_workers
        dims, ag = self._spec.dims, self.agent
        self._upload_batch()
        slot.theta_prev.copy_(slot.theta)
        self._draw_offsets()
        gt = self._grad_table()
        rm = W > 1 and gt.dtype == torch.float16
        self._rm_live = rm
        BC = self._bc
        if rm:
            R, N = self._rm_buffers()
            ret_p, ret_m, nov_p, nov_m = R[self.rank, 0], R[self.rank, 1], N[self.rank, 0], N[self.rank, 1]
        else:
            R, N = self._returns, self._novelty
            ret_p, ret_m = R[pb: pb + pl], R[pairs + pb: pairs + pb + pl]
            nov_p, nov_m = N[pb: pb + pl], N[pairs + pb: pairs + pb + pl]
        self._eval_fns()[0](dims, slot.theta, self._table, self._offsets, self._order, pl, self.sigma,
                            self._obs, self._tgt, ret_p, ret_m,
                            BC[pb: pb + pl], BC[pairs + pb: pairs + pb + pl], ag.bc_obs, ag.bc_dim,
                            **self._mlp_kw(slot))
        be.knn_novelty(BC[pb: pb + pl], self._arch_dev, self.k, nov_p)
        be.knn_novelty(BC[pairs + pb: pairs + pb + pl], self._arch_dev, self.k, nov_m)
        self._update_step(slot, R, N, np.float32(self._w_rew()), np.float32(self._w_nov()), rm)
        # _after_optimize (estorch.py:427-432 / :650-662): rollout of the updated
        # policy, archive append, best tracking, NSRA schedule (host scalars)
        self._centre_bc(slot)
        self._after_update(slot)

    def _after_update(self, slot):
        """The host side of ``_after_optimize`` once theta's rollout is in ``self._episode`` /
        ``self._bc_center[0]``: archive append, best tracking, NSRA schedule."""
        episode = float(self._episode.item())
        self._archive.append(self._bc_center[0].cpu().numpy().copy())
        self.episode_reward = episode
        improved = episode > self._best_host
        if improved:
            self._best_host = episode
            slot.best_theta.copy_(slot.theta)
            self._best_slot = slot
        self.best_reward = self._best_host
        self._on_after_optimize(improved)

    def _on_after_optimize(self, improved):
        pass


class NSR_ES(NS_ES):
    """NSR-ES: average of reward and novelty centred ranks (estorch.py:475-549)."""
    _W_REW, _W_NOV = 0.5, 0.5


class NSRA_ES(NS_ES):
    """NSRA-ES: adaptive blend ``w*c(reward) + (1-w)*c(novelty)`` with the
    weight schedule of estorch.py:650-662.  As in the reference (estorch.py:637)
    ``weight_delta`` is fixed at 0.05 regardless of the constructor argument."""

    def __init__(self, policy, agent, optimizer, population_size, sigma=0.01,
                 meta_population_size=3, k=10, min_weight=0.0, weight_t=50,
                 weight_delta=0.05, device=torch.device("cpu"),
                 policy_kwargs={}, agent_kwargs={}, optimizer_kwargs={}, **engine_kwargs):
        super().__init__(policy=policy, agent=agent, optimizer=optimizer,
                         population_size=population_size, sigma=sigma,
                         meta_population_size=meta_population_size, k=k, device=device,
                         policy_kwargs=policy_kwargs, agent_kwargs=agent_kwargs,
                         optimizer_kwargs=optimizer_kwargs, **engine_kwargs)
        self.weight = 1.0
        self.min_weight = min_weight
        self.weight_t = weight_t
        self.weight_delta = 0.05                                      # estorch.py:637
        self.t = 0

    def _w_rew(self):
        return self.weight

    def _w_nov(self):
        return 1.0 - self.weight

    def _schedule(self, improved):
        if improved:                                                  # estorch.py:653-657
            self.weight = min(self.weight + self.weight_delta, 1.0)
            self.t = 0
        else:                                                         # :658-662
            self.t += 1
            if self.t >= self.weight_t:
                self.weight = max(self.weight - self.weight_delta, self.min_weight)
                self.t = 0

    @_builtin
    def _after_optimize(self, policy):
        self.episode_reward, bc = self.agent.rollout(policy)
        self._archive.append(bc)
        improved = self.episode_reward > self.best_reward
        if improved:
            self.best_reward = self.episode_reward
            self.best_policy_dict = copy.deepcopy(policy.state_dict())
        self._schedule(improved)

    def _on_after_optimize(self, improved):
        self._schedule(improved)
