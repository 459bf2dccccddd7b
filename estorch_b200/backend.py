"""CudaBackend -- the single product implementation of the kernel interface.

A 1:1 pythonic mirror of include/estk.h: every method takes torch tensors that
live on ``self.device`` (PyTorch is only the allocator / stream provider here),
checks dtype / contiguity, and enqueues the C-ABI call on torch's current
stream.  There is no CPU implementation in the product; tests that exercise the
host logic without a GPU inject their own stand-in built on ``oracle/``.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
import torch

from . import _capi

STATE_BYTES = C.sizeof(_capi.EstkState)
STATE_DTYPE = np.dtype([("generation", "<i8"), ("adam_step", "<i8"), ("episode_reward", "<f4"),
                        ("best_reward", "<f4"), ("improved", "<i4"), ("reserved", "<i4")])
assert STATE_DTYPE.itemsize == STATE_BYTES == 32


def new_state(device) -> torch.Tensor:
    """A zeroed ``estk_state`` with best_reward = -inf (estorch.py:145)."""
    host = np.zeros(1, dtype=STATE_DTYPE)
    host["best_reward"] = -np.inf
    return torch.from_numpy(host.view(np.uint8).copy()).to(device)


def read_state(state: torch.Tensor) -> dict:
    rec = state.detach().cpu().numpy().view(STATE_DTYPE)[0]
    return {k: rec[k].item() for k in STATE_DTYPE.names}


def write_state(state: torch.Tensor, **fields):
    rec = state.detach().cpu().numpy().copy().view(STATE_DTYPE)
    for k, v in fields.items():
        rec[k] = v
    state.copy_(torch.from_numpy(rec.view(np.uint8).copy()))


def mlp_desc(dims: Sequence[int], act: int = 0, steps: int = 0) -> _capi.EstkMlpDesc:
    """``act``: the ``estk_mlp_desc.activation`` code (``MLPSpec.act``; 0 = ReLU hidden, identity output).
    ``steps``: T of a recurrent sequence evaluate, stored in ``dims[3]`` after ``dims = (in, H, out)``."""
    if not (2 <= len(dims) <= _capi.ESTK_MAX_LAYERS + 1):
        raise ValueError(f"MLP with {len(dims) - 1} Linear layers is outside 1..{_capi.ESTK_MAX_LAYERS}")
    d = _capi.EstkMlpDesc()
    d.n_layers = len(dims) - 1
    for i, w in enumerate(dims):
        d.dims[i] = int(w)
    if steps:
        if len(dims) != 3:
            raise ValueError("steps belongs to a recurrent policy's dims = (in, H, out)")
        d.dims[3] = int(steps)
    d.activation = int(act)
    return d


def cnn_desc(spec, code: int) -> _capi.EstkMlpDesc:
    """The ``estk_mlp_desc`` of a convolutional policy: ``spec`` is a ``CNNSpec`` or its packed ``dims``
    (``ESTK_CNN_INPUT``, one ``ESTK_CNN_CONV`` per conv, the Linear widths); ``code`` the activation code,
    whose bits 24-31 hold n_conv."""
    dims = spec.dims if hasattr(spec, "dims") else tuple(spec)
    if not (code >> _capi.ESTK_CNN_SHIFT) & 0xff:
        raise ValueError(f"activation code {code:#x} has no conv layers in bits 24-31")
    d = _capi.EstkMlpDesc()
    d.n_layers = len(dims) - 1
    if not 1 <= d.n_layers <= _capi.ESTK_MAX_LAYERS:
        raise ValueError(f"CNN with {len(dims) - 1} layers is outside 1..{_capi.ESTK_MAX_LAYERS}")
    for i, w in enumerate(dims):
        d.dims[i] = C.c_int32(int(w)).value
    d.activation = C.c_int32(int(code)).value
    return d


def cnn_shapes(dims, code):
    """((c, h, w), out) of the packed ``dims`` and activation ``code`` of a convolutional policy."""
    dims = [int(x) & 0xffffffff for x in dims]
    c, h, w = dims[0] & 1023, (dims[0] >> 10) & 1023, (dims[0] >> 20) & 1023
    return (c, h, w), dims[-1]


def adam_desc(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, clamp=1.0) -> _capi.EstkAdamDesc:
    a = _capi.EstkAdamDesc()
    a.lr, a.beta1, a.beta2, a.eps = float(lr), float(betas[0]), float(betas[1]), float(eps)
    a.weight_decay, a.clamp = float(weight_decay), float(clamp)
    return a


# eval_precision -> (ESTK_PREC_* code, dtype of its 16-bit theta16 / table16 buffers)
_PRECISIONS = {"fp32": (_capi.ESTK_PREC_FP32, None), "f16": (_capi.ESTK_PREC_F16, torch.float16),
               "bf16": (_capi.ESTK_PREC_BF16, None), "bf16s": (_capi.ESTK_PREC_BF16S, torch.bfloat16),
               "f16_any": (_capi.ESTK_PREC_F16_ANY, torch.float16)}


class CudaBackend:
    """Kernel interface over libestk.so on one CUDA device."""

    name = "cuda"

    def __init__(self, device: Optional[torch.device] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("estorch_b200 needs a CUDA device (H100, sm_90a); "
                               "torch.cuda.is_available() is False and there is no CPU fallback")
        self.lib = _capi.load()
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"CudaBackend needs a cuda device, got {device}")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = device
        torch.cuda.set_device(device)
        ctx = C.c_void_p()
        _capi.check(self.lib.estk_ctx_create(device.index, C.byref(ctx)), "estk_ctx_create")
        self._ctx = ctx
        sm, mj, mn = C.c_int(), C.c_int(), C.c_int()
        _capi.check(self.lib.estk_ctx_info(ctx, C.byref(sm), C.byref(mj), C.byref(mn)), "estk_ctx_info")
        self.sm_count, self.cc = sm.value, (mj.value, mn.value)
        self.launches = 0  # kernels of OUR library enqueued through this backend

    def __del__(self):
        ctx = getattr(self, "_ctx", None)
        if ctx:
            try:
                self.peer_close_all()
                self.lib.estk_ctx_destroy(ctx)
            except Exception:
                pass
            self._ctx = None

    # ---------------------------------------------------------------- helpers
    def _ptr(self, t: Optional[torch.Tensor], dtype=None, name="tensor"):
        if t is None or isinstance(t, C.c_void_p):   # no buffer, or a pointer made (and checked) by the caller
            return t
        if t.device != self.device:
            raise ValueError(f"{name} is on {t.device}, backend is on {self.device}")
        if dtype is not None and t.dtype != dtype:
            raise ValueError(f"{name} has dtype {t.dtype}, expected {dtype}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
        return C.c_void_p(t.data_ptr())

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def alloc(self, *shape, dtype=torch.float32):
        return torch.empty(*shape, dtype=dtype, device=self.device)

    def zeros(self, *shape, dtype=torch.float32):
        return torch.zeros(*shape, dtype=dtype, device=self.device)

    # ---------------------------------------------------------------- noise
    def fill_noise_table(self, table: torch.Tensor, seed: int):
        _capi.check(self.lib.estk_fill_noise_table(self._ctx, self._ptr(table, torch.float32, "table"),
                                                   table.numel(), seed & (2**64 - 1), self._stream()),
                    "estk_fill_noise_table")
        self.launches += 1

    def make_offsets(self, seed, state, gen_host, pair_begin, pairs, table_len, n, offsets_out,
                     order_out=None):
        _capi.check(self.lib.estk_make_offsets(
            self._ctx, seed & (2**64 - 1), self._ptr(state, torch.uint8, "state"), int(gen_host),
            int(pair_begin), int(pairs), int(table_len), int(n),
            self._ptr(offsets_out, torch.int64, "offsets_out"),
            self._ptr(order_out, torch.int32, "order_out"), self._stream()), "estk_make_offsets")
        self.launches += 1

    def perturb_rows(self, theta, table, offsets, pairs, sigma, member_begin, member_count,
                     rows_out=None, eps_out=None):
        _capi.check(self.lib.estk_perturb_rows(
            self._ctx, self._ptr(theta, torch.float32, "theta"), theta.numel(),
            self._ptr(table, torch.float32, "table"), self._ptr(offsets, torch.int64, "offsets"),
            int(pairs), float(sigma), int(member_begin), int(member_count),
            self._ptr(rows_out, torch.float32, "rows_out"), self._ptr(eps_out, torch.float32, "eps_out"),
            self._stream()), "estk_perturb_rows")
        self.launches += 1

    # ---------------------------------------------------------------- minibatches
    def sample_batch(self, seed, state, gen_host, obs_src, obs_dst, tgt_src, tgt_dst, index_out=None):
        """Generation g's minibatch of the dataset ``obs_src`` ``[N, ...]`` / ``tgt_src`` ``[N, ...]`` into
        ``obs_dst`` ``[B, ...]`` / ``tgt_dst`` ``[B, ...]`` (estk_sample_batch; ``batch_indices`` states the rows);
        g = ``gen_host`` plus the generation in ``state`` (None: ``gen_host`` alone).  ``index_out`` (int64
        ``[B]``, optional) receives the row indices."""
        N, B = int(obs_src.shape[0]), int(obs_dst.shape[0])
        if obs_src.dim() < 1 or tuple(obs_dst.shape[1:]) != tuple(obs_src.shape[1:]) or \
                tuple(tgt_src.shape[:1]) != (N,) or tuple(tgt_dst.shape) != (B,) + tuple(tgt_src.shape[1:]):
            raise ValueError(f"sample_batch: obs {tuple(obs_src.shape)} -> {tuple(obs_dst.shape)}, target "
                             f"{tuple(tgt_src.shape)} -> {tuple(tgt_dst.shape)} are not [N, ...] -> [B, ...]")
        if index_out is not None and tuple(index_out.shape) != (B,):
            raise ValueError(f"sample_batch: index_out {tuple(index_out.shape)}, expected [{B}]")
        _capi.check(self.lib.estk_sample_batch(
            self._ctx, int(seed) & (2**64 - 1), self._ptr(state, torch.uint8, "state"), int(gen_host), N, B,
            self._ptr(obs_src, torch.float32, "obs_src"), obs_src[0].numel() if N else 0,
            self._ptr(obs_dst, torch.float32, "obs_dst"), self._ptr(tgt_src, torch.float32, "tgt_src"),
            tgt_src[0].numel() if N else 0, self._ptr(tgt_dst, torch.float32, "tgt_dst"),
            self._ptr(index_out, torch.int64, "index_out"), self._stream()), "estk_sample_batch")
        self.launches += 1

    # ---------------------------------------------------------------- evaluate
    def _precision(self, precision):
        """ESTK_PREC_* code and the dtype of the 16-bit buffers (theta16 / table16) of an evaluate precision."""
        try:
            return _PRECISIONS[precision]
        except KeyError:
            raise ValueError(f"unknown precision {precision!r}") from None

    def eval_supports_bf16(self, dims, B, act=0) -> bool:
        d = mlp_desc(dims, act)
        return bool(self.lib.estk_eval_mlp_supported(C.byref(d), _capi.ESTK_PREC_BF16, int(B)))

    def eval_supports_f16(self, dims, B, act=0) -> bool:
        d = mlp_desc(dims, act)
        return bool(self.lib.estk_eval_mlp_supported(C.byref(d), _capi.ESTK_PREC_F16, int(B)))

    def eval_supports_f16_any(self, dims, B, act=0) -> bool:
        """``"f16_any"``: the F16 arithmetic for every MLP shape (False only for an invalid code or B < 1)."""
        d = mlp_desc(dims, act)
        return bool(self.lib.estk_eval_mlp_supported(C.byref(d), _capi.ESTK_PREC_F16_ANY, int(B)))

    def eval_supports_tf32_cnn(self, dims, B, act=0) -> bool:
        """``"tf32"`` for a convolutional policy (``dims`` its packed descriptor or ``CNNSpec``, ``act`` its code
        with n_conv): every valid descriptor whose largest layer output is at most 2**26 floats per image."""
        try:
            d = cnn_desc(dims, act)
        except ValueError:
            return False
        return bool(self.lib.estk_eval_cnn_tf32_supported(C.byref(d), int(B)))

    def shadow_f16(self, src, dst, check=True) -> int:
        """dst (float16, same numel) = src; returns how many entries were NOT exactly
        representable (0 for tables made by fill_noise_table).  ``check`` reads the
        counter back (one host synchronisation; setup time only)."""
        cnt = torch.zeros(1, dtype=torch.int64, device=self.device) if check else None
        _capi.check(self.lib.estk_shadow_f16(self._ctx, self._ptr(src, torch.float32, "src"),
                                             self._ptr(dst, torch.float16, "dst"), src.numel(),
                                             self._ptr(cnt, torch.int64, "inexact"), self._stream()),
                    "estk_shadow_f16")
        self.launches += 1
        return int(cnt.item()) if check else 0

    def shadow_bf16(self, src, dst):
        """dst (int16/bfloat16 storage, same numel) = bf16(src)."""
        _capi.check(self.lib.estk_shadow_bf16(self._ctx, self._ptr(src, torch.float32, "src"),
                                              self._ptr(dst, torch.bfloat16, "dst"), src.numel(), self._stream()),
                    "estk_shadow_bf16")
        self.launches += 1

    def _eval_mlp(self, what, d, code, B, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus,
                  ret_minus, bc_plus, bc_minus, bc_obs, bc_dim, dt16=None, theta16=None, table16=None, centre_out=None,
                  launches=1):
        """One estk_eval_mlp call on the current stream: ``d`` the descriptor, ``code`` the ESTK_PREC_* code,
        ``dt16`` the dtype of theta16 / table16; ``what`` names the call in an error."""
        _capi.check(self.lib.estk_eval_mlp(
            self._ctx, C.byref(d), code, self._ptr(theta, torch.float32, "theta"),
            self._ptr(theta16, dt16, "theta16"), self._ptr(table, torch.float32, "table"),
            self._ptr(table16, dt16, "table16"), self._ptr(offsets, torch.int64, "offsets"),
            self._ptr(order, torch.int32, "order"), int(pairs), float(sigma), self._ptr(obs, torch.float32, "obs"),
            self._ptr(target, torch.float32, "target"), int(B),
            self._ptr(ret_plus, torch.float32, "ret_plus"), self._ptr(ret_minus, torch.float32, "ret_minus"),
            self._ptr(bc_plus, torch.float32, "bc_plus"), self._ptr(bc_minus, torch.float32, "bc_minus"),
            int(bc_obs), int(bc_dim), self._ptr(centre_out, torch.float32, "centre_out"), self._stream()), what)
        self.launches += launches

    def eval_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, target,
                 ret_plus, ret_minus, bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32",
                 theta16=None, table16=None, centre_out=None, act=0):
        """Population evaluate (estk_eval_mlp); ``offsets`` None = the centre evaluation into ``ret_plus[0]``."""
        code, dt16 = self._precision(precision)
        d = mlp_desc(dims, act)
        if obs.shape != (obs.shape[0], dims[0]) or target.shape != (obs.shape[0], dims[-1]):
            raise ValueError(f"obs {tuple(obs.shape)} / target {tuple(target.shape)} do not match dims {list(dims)}")
        # "f16_any" off the cluster kernel's shapes: the observation split, then the streamed kernel
        launches = 2 if precision == "f16_any" and not self.eval_supports_f16(dims, obs.shape[0], act) else 1
        self._eval_mlp(f"estk_eval_mlp[{precision}]", d, code, obs.shape[0], theta, table, offsets, order, pairs,
                       sigma, obs, target, ret_plus, ret_minus, bc_plus, bc_minus, bc_obs, bc_dim, dt16=dt16,
                       theta16=theta16, table16=table16, centre_out=centre_out, launches=launches)

    def eval_mlp_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0,
                        precision="fp32", theta16=None, act=0):
        """Unperturbed policy: ``ret_out[0]`` = return of theta, ``bc_out`` its behaviour characteristic."""
        self.eval_mlp(dims, theta, None, None, None, 1, 0.0, obs, target, ret_out, None, bc_out, None, bc_obs, bc_dim,
                      precision=precision, theta16=theta16, act=act)

    def act_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, out, act=0, table16=None):
        """Every perturbed policy's outputs on its own observations (estk_eval_mlp with ESTK_ACTIONS, fp32).
        Population: ``obs`` ``[2*pairs, B, in]`` -> ``out`` ``[2*pairs, B, out]``, rows ``< pairs`` the + members
        of the local pairs, the rest their mirrors.  ``offsets`` None = the centre: ``obs`` / ``out``
        ``[1, B, ...]`` for theta.  ``act``: the policy's hidden / output code (ESTK_ACTIONS is added here);
        ``table16``: the exact fp16 copy of ``table``, read instead of it."""
        self._act(dims, 0, "estk_eval_mlp[actions]", theta, table, offsets, order, pairs, sigma, obs, out, act,
                  table16)

    def act_rnn(self, dims, theta, table, offsets, order, pairs, sigma, obs, out, act, table16=None):
        """One step of every perturbed recurrent policy (estk_eval_mlp with ESTK_CELL_GRU / ESTK_CELL_LSTM and
        ESTK_ACTIONS, fp32).  ``dims`` = (in, H, out); ``act``: the cell | output code (ESTK_ACTIONS is added
        here).  Population: ``obs`` ``[2*pairs, B, in + S]`` (x, then the state h, and c for LSTM) ->
        ``out`` ``[2*pairs, B, out + S]`` (y, then h', and c'), S = H (GRU) or 2H (LSTM); ``offsets`` None =
        the centre, ``[1, B, ...]`` for theta.  ``table16``: the exact fp16 copy of ``table``, read instead of it."""
        din, H, dout = (int(d) for d in dims)
        S = H if (int(act) & 0xff) == _capi.ESTK_CELL_GRU else 2 * H
        self._act(dims, S, "estk_eval_mlp[recurrent actions]", theta, table, offsets, order, pairs, sigma, obs, out,
                  act, table16)

    def _act(self, dims, S, what, theta, table, offsets, order, pairs, sigma, obs, out, act, table16):
        """act_mlp (``S`` = 0) and act_rnn (``S`` the width of the recurrent state after x in obs and y in out)."""
        M = 1 if offsets is None else 2 * int(pairs)
        if obs.dim() != 3 or tuple(obs.shape) != (M, obs.shape[1], dims[0] + S) or \
                tuple(out.shape) != (M, obs.shape[1], dims[-1] + S):
            policy = f"the recurrent policy {[int(w) for w in dims]} (state width {S})" if S else f"dims {list(dims)}"
            raise ValueError(f"obs {tuple(obs.shape)} / out {tuple(out.shape)} do not match {policy} for {M} members")
        d = mlp_desc(dims, (int(act) & 0xffff) | _capi.ESTK_ACTIONS)
        B, per = int(obs.shape[1]), int(obs.shape[1]) * (int(dims[-1]) + S)
        minus = None if offsets is None else C.c_void_p(out.data_ptr() + int(pairs) * per * out.element_size())
        self._eval_mlp(what, d, _capi.ESTK_PREC_FP32, B, theta, None if table16 is not None else table, offsets,
                       order, pairs, sigma, obs, None, None, None, self._ptr(out, torch.float32, "out"), minus, B, per,
                       dt16=torch.float16, table16=table16)

    def eval_rnn_seq(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                     bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", act=0):
        """Sequence evaluate of a recurrent policy (estk_eval_mlp with ESTK_CELL_GRU / ESTK_CELL_LSTM and a
        return, fp32): ``dims`` = (in, H, out), ``obs`` ``[B, T, in]``, ``target`` ``[B, T, out]``; ``act``: the
        cell | output | loss code.  The arguments are ``eval_mlp``'s fp32 ones, so the engine calls either the
        same way; ``precision`` other than "fp32" is refused by the library."""
        code, _dt16 = self._precision(precision)
        B, T = int(obs.shape[0]), int(obs.shape[1]) if obs.dim() == 3 else 0
        if obs.dim() != 3 or tuple(obs.shape) != (B, T, dims[0]) or tuple(target.shape) != (B, T, dims[-1]):
            raise ValueError(f"obs {tuple(obs.shape)} / target {tuple(target.shape)} do not match the recurrent "
                             f"policy {list(dims)}: expected [B, T, {dims[0]}] / [B, T, {dims[-1]}]")
        self._eval_mlp(f"estk_eval_mlp[recurrent sequence, {precision}]", mlp_desc(dims, act, steps=T), code, B,
                       theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus, bc_plus,
                       bc_minus, bc_obs, bc_dim)

    def eval_rnn_seq_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0,
                            precision="fp32", act=0):
        """Unperturbed recurrent policy: ``ret_out[0]`` = return of theta, ``bc_out`` its behaviour characteristic."""
        self.eval_rnn_seq(dims, theta, None, None, None, 1, 0.0, obs, target, ret_out, None, bc_out, None, bc_obs,
                          bc_dim, precision=precision, act=act)

    def eval_cnn(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                 bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", act=0):
        """Fixed-batch evaluate of a convolutional policy (estk_eval_mlp with n_conv in bits 24-31 of ``act``,
        fp32): ``dims`` the packed descriptor (``CNNSpec.dims``, or the spec itself), ``obs`` ``[B, c, h, w]``,
        ``target`` ``[B, out]``.  The arguments are ``eval_mlp``'s fp32 ones, so the engine calls either the same
        way.  ``precision="tf32"``: the same evaluate on TF32 tensor cores (estk_eval_cnn_tf32); any other
        precision but "fp32" is refused by the library."""
        code = None if precision == "tf32" else self._precision(precision)[0]
        d = cnn_desc(dims, act)
        (c, h, w), out = cnn_shapes([d.dims[i] for i in range(d.n_layers + 1)], act)
        B = int(obs.shape[0])
        if tuple(obs.shape) != (B, c, h, w) or tuple(target.shape) != (B, out):
            raise ValueError(f"obs {tuple(obs.shape)} / target {tuple(target.shape)} do not match the convolutional "
                             f"policy: expected [B, {c}, {h}, {w}] / [B, {out}]")
        if code is None:
            _capi.check(self.lib.estk_eval_cnn_tf32(
                self._ctx, C.byref(d), self._ptr(theta, torch.float32, "theta"), self._ptr(table, torch.float32, "table"),
                self._ptr(offsets, torch.int64, "offsets"), self._ptr(order, torch.int32, "order"), int(pairs),
                float(sigma), self._ptr(obs, torch.float32, "obs"), self._ptr(target, torch.float32, "target"), B,
                self._ptr(ret_plus, torch.float32, "ret_plus"), self._ptr(ret_minus, torch.float32, "ret_minus"),
                self._ptr(bc_plus, torch.float32, "bc_plus"), self._ptr(bc_minus, torch.float32, "bc_minus"),
                int(bc_obs), int(bc_dim), self._stream()), "estk_eval_cnn_tf32")
            self.launches += 1
            return
        self._eval_mlp(f"estk_eval_mlp[convolutional, {precision}]", d, code, B, theta, table, offsets, order, pairs,
                       sigma, obs, target, ret_plus, ret_minus, bc_plus, bc_minus, bc_obs, bc_dim)

    def eval_cnn_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0,
                        precision="fp32", act=0):
        """Unperturbed convolutional policy: ``ret_out[0]`` = return of theta, ``bc_out`` its behaviour
        characteristic."""
        self.eval_cnn(dims, theta, None, None, None, 1, 0.0, obs, target, ret_out, None, bc_out, None, bc_obs,
                      bc_dim, precision=precision, act=act)

    def act_cnn(self, dims, theta, table, offsets, order, pairs, sigma, obs, out, act):
        """Every perturbed convolutional policy's outputs on its own images (estk_act_cnn, fp32).  ``dims`` the
        packed descriptor (``CNNSpec.dims``, or the spec itself); ``act`` the hidden | output | n_conv code
        (ESTK_ACTIONS is added here).  Population: ``obs`` ``[2*pairs, B, c, h, w]`` -> ``out``
        ``[2*pairs, B, out]``, rows ``< pairs`` the + members of the local pairs, the rest their mirrors.
        ``offsets`` None = the centre: ``obs`` / ``out`` ``[1, B, ...]`` for theta."""
        d = cnn_desc(dims, (int(act) & 0xff00ffff) | _capi.ESTK_ACTIONS)
        (c, h, w), n_out = cnn_shapes([d.dims[i] for i in range(d.n_layers + 1)], act)
        M = 1 if offsets is None else 2 * int(pairs)
        B = int(obs.shape[1]) if obs.dim() == 5 else -1
        if obs.dim() != 5 or tuple(obs.shape) != (M, B, c, h, w) or tuple(out.shape) != (M, B, n_out):
            raise ValueError(f"obs {tuple(obs.shape)} / out {tuple(out.shape)} do not match the convolutional policy "
                             f"for {M} members: expected [{M}, B, {c}, {h}, {w}] / [{M}, B, {n_out}]")
        minus = None if offsets is None else C.c_void_p(out.data_ptr() + int(pairs) * B * n_out * out.element_size())
        _capi.check(self.lib.estk_act_cnn(
            self._ctx, C.byref(d), self._ptr(theta, torch.float32, "theta"), self._ptr(table, torch.float32, "table"),
            self._ptr(offsets, torch.int64, "offsets"), self._ptr(order, torch.int32, "order"), int(pairs),
            float(sigma), self._ptr(obs, torch.float32, "obs"), B, self._ptr(out, torch.float32, "out"), minus,
            self._stream()), "estk_act_cnn")
        self.launches += 1

    def conv_scratch_bytes(self, ref_batch, B, precision="fp32") -> int:
        return int(self.lib.estk_eval_conv_vbn_scratch_bytes(self._ctx, self._precision(precision)[0], int(ref_batch),
                                                             int(B)))

    def eval_conv_vbn(self, n_actions, theta, table, offsets, order, pairs, sigma, xref, obs, target,
                      ret_plus, ret_minus, scratch, precision="fp32", table16=None):
        """Conv + VirtualBatchNorm policy (examples/atari.py:14-37); offsets None = centre.
        precision "f16": the tensor-core kernel (needs table16 with offsets, and a scratch of
        conv_scratch_bytes(R, B, "f16") bytes)."""
        code, dt16 = self._precision(precision)
        _capi.check(self.lib.estk_eval_conv_vbn(
            self._ctx, code, int(n_actions), self._ptr(theta, torch.float32, "theta"),
            self._ptr(table, torch.float32, "table"), self._ptr(table16, dt16, "table16"),
            self._ptr(offsets, torch.int64, "offsets"), self._ptr(order, torch.int32, "order"), int(pairs),
            float(sigma), self._ptr(xref, torch.float32, "xref"), int(xref.shape[0]),
            self._ptr(obs, torch.float32, "obs"), self._ptr(target, torch.float32, "target"), int(obs.shape[0]),
            self._ptr(ret_plus, torch.float32, "ret_plus"), self._ptr(ret_minus, torch.float32, "ret_minus"),
            self._ptr(scratch, torch.uint8, "scratch"), scratch.numel(), self._stream()),
            f"estk_eval_conv_vbn[{precision}]")
        self.launches += 1

    def act_conv_vbn(self, n_actions, theta, table, offsets, order, pairs, sigma, xref, obs, out, stats,
                     table16=None):
        """The conv + VirtualBatchNorm policy's action mode (estk_eval_conv_vbn with ESTK_ACTIONS, fp32).
        ``xref`` ``[R, 4, 84, 84]`` (or None): compute every member's VBN statistics into ``stats`` (float32,
        ``[members, ESTK_CONV_VBN_STATS_FLOATS]``).  ``obs`` (or None): every member's outputs on its own frames
        from the statistics in ``stats``; population ``obs`` ``[2*pairs, B, 4, 84, 84]`` -> ``out``
        ``[2*pairs, B, A]`` (rows ``< pairs`` the + members of the local pairs, the rest their mirrors);
        ``offsets`` None = the centre, ``obs`` / ``out`` ``[1, B, ...]`` for theta.  ``table16``: the exact fp16
        copy of ``table``, read instead of it."""
        M = 1 if offsets is None else 2 * int(pairs)
        A = int(n_actions)
        if tuple(stats.shape) != (M, _capi.ESTK_CONV_VBN_STATS_FLOATS):
            raise ValueError(f"stats {tuple(stats.shape)}, expected [{M}, {_capi.ESTK_CONV_VBN_STATS_FLOATS}]")
        B, per = 1, 0
        if obs is not None:
            B = int(obs.shape[1]) if obs.dim() == 5 else -1
            if obs.dim() != 5 or tuple(obs.shape) != (M, B, 4, 84, 84) or tuple(out.shape) != (M, B, A):
                raise ValueError(f"obs {tuple(obs.shape)} / out {tuple(out.shape)}, expected [{M}, B, 4, 84, 84] / "
                                 f"[{M}, B, {A}]")
            per = B * A
        t32 = None if table16 is not None else table
        _capi.check(self.lib.estk_eval_conv_vbn(
            self._ctx, _capi.ESTK_PREC_FP32, A | _capi.ESTK_ACTIONS, self._ptr(theta, torch.float32, "theta"),
            self._ptr(t32, torch.float32, "table"), self._ptr(table16, torch.float16, "table16"),
            self._ptr(offsets, torch.int64, "offsets"), self._ptr(order, torch.int32, "order"), int(pairs),
            float(sigma), self._ptr(xref, torch.float32, "xref"), 0 if xref is None else int(xref.shape[0]),
            self._ptr(obs, torch.float32, "obs"), None, B,
            None if obs is None else self._ptr(out, torch.float32, "out"),
            None if obs is None or offsets is None else C.c_void_p(out.data_ptr() + int(pairs) * per * 4),
            self._ptr(stats, torch.float32, "stats"), stats.numel() * 4, self._stream()),
            "estk_eval_conv_vbn[actions]")
        self.launches += (xref is not None) + (obs is not None)

    def track_best(self, state, reward, theta, best_theta):
        _capi.check(self.lib.estk_track_best(
            self._ctx, self._ptr(state, torch.uint8, "state"), self._ptr(reward, torch.float32, "reward"),
            self._ptr(theta, torch.float32, "theta"), self._ptr(best_theta, torch.float32, "best_theta"),
            theta.numel(), self._stream()), "estk_track_best")
        self.launches += 1

    # ---------------------------------------------------------------- rank + grad + Adam
    def _tables(self, table):
        """(table, table16) pointers of estk_rank_grad*: ``table`` is float32, or float16 = the exact 16-bit
        copy (half the bytes, same result)."""
        if table.dtype == torch.float16:
            return None, self._ptr(table, torch.float16, "table16")
        return self._ptr(table, torch.float32, "table"), None

    def rank_grad_adam(self, returns, novelty, w_rew, w_nov, P, table, offsets, order, theta, m, v,
                       state, adam, ranks_out=None, ranks2_out=None, grad_out=None):
        _capi.check(self.lib.estk_rank_grad_adam(
            self._ctx, self._ptr(returns, torch.float32, "returns"),
            self._ptr(novelty, torch.float32, "novelty"), float(w_rew), float(w_nov), int(P), *self._tables(table),
            self._ptr(offsets, torch.int64, "offsets"), self._ptr(order, torch.int32, "order"), theta.numel(),
            self._ptr(theta, torch.float32, "theta"), self._ptr(m, torch.float32, "m"),
            self._ptr(v, torch.float32, "v"), self._ptr(state, torch.uint8, "state"), C.byref(adam),
            self._ptr(ranks_out, torch.int32, "ranks_out"), self._ptr(ranks2_out, torch.int32, "ranks2_out"),
            self._ptr(grad_out, torch.float32, "grad_out"), self._stream()), "estk_rank_grad_adam")
        self.launches += 1

    def rank_grad(self, returns, novelty, w_rew, w_nov, P, table, offsets, order, pair_begin,
                  pairs_local, n, grad_sum_out, ranks_out=None, ranks2_out=None, world=1):
        """``world > 1`` declares rank-major returns ``[world][2][pairs/world]``."""
        _capi.check(self.lib.estk_rank_grad(
            self._ctx, self._ptr(returns, torch.float32, "returns"), self._ptr(novelty, torch.float32, "novelty"),
            float(w_rew), float(w_nov), int(P), int(world), *self._tables(table),
            self._ptr(offsets, torch.int64, "offsets"), self._ptr(order, torch.int32, "order"), int(pair_begin),
            int(pairs_local), int(n), self._ptr(grad_sum_out, torch.float32, "grad_sum_out"),
            self._ptr(ranks_out, torch.int32, "ranks_out"), self._ptr(ranks2_out, torch.int32, "ranks2_out"),
            self._stream()), "estk_rank_grad")
        self.launches += 1

    # ---------------------------------------------------------------- peer memory (CUDA IPC)
    def peer_alloc(self, nbytes: int):
        """Zero-filled device memory another process of this node can map: ``(pointer, 64-byte handle)``."""
        ptr, handle = C.c_void_p(), C.create_string_buffer(64)
        _capi.check(self.lib.estk_peer_alloc(self._ctx, int(nbytes), C.byref(ptr), handle), "estk_peer_alloc")
        self._peer_owned = getattr(self, "_peer_owned", []) + [ptr.value]
        return ptr.value, bytes(handle.raw)

    def peer_open(self, handle: bytes) -> int:
        ptr = C.c_void_p()
        _capi.check(self.lib.estk_peer_open(self._ctx, C.create_string_buffer(handle, 64), C.byref(ptr)), "estk_peer_open")
        self._peer_mapped = getattr(self, "_peer_mapped", []) + [ptr.value]
        return ptr.value

    def peer_close_all(self):
        """Unmap the peers' workspaces (when no kernel of this process uses them any more)."""
        for ptr in getattr(self, "_peer_mapped", []):
            self.lib.estk_peer_close(self._ctx, C.c_void_p(ptr))
        self._peer_mapped = []

    def peer_free_all(self):
        """Free this process's own workspaces -- only after EVERY peer unmapped them (a barrier in between:
        ``estorch._shutdown_dist``).  Never called from ``__del__``: 8 MB per instance wait for process exit."""
        for ptr in getattr(self, "_peer_owned", []):
            self.lib.estk_peer_free(self._ctx, C.c_void_p(ptr))
        self._peer_owned = []

    def xr_workspace_bytes(self, n: int) -> int:
        return int(self.lib.estk_xr_workspace_bytes(int(n)))

    def rank_grad_xr_adam(self, returns, novelty, w_rew, w_nov, P, world, rank, table16, offsets, order, pair_begin,
                          pairs_local, peer_ptrs, theta, m, v, state, adam, ranks_out=None, ranks2_out=None,
                          grad_out=None):
        """Rank + partial gradient + cross-GPU sum over peer memory + Adam in one launch (estk.h).
        ``returns`` / ``novelty`` rank-major; ``peer_ptrs`` = every rank's workspace as mapped here."""
        arr = (C.c_void_p * world)(*[C.c_void_p(x) for x in peer_ptrs])
        _capi.check(self.lib.estk_rank_grad_xr_adam(
            self._ctx, self._ptr(returns, torch.float32, "returns"), self._ptr(novelty, torch.float32, "novelty"),
            float(w_rew), float(w_nov), int(P), int(world), int(rank), self._ptr(table16, torch.float16, "table16"),
            self._ptr(offsets, torch.int64, "offsets"), self._ptr(order, torch.int32, "order"), int(pair_begin),
            int(pairs_local), theta.numel(), arr, self._ptr(theta, torch.float32, "theta"),
            self._ptr(m, torch.float32, "m"), self._ptr(v, torch.float32, "v"), self._ptr(state, torch.uint8, "state"),
            C.byref(adam), self._ptr(ranks_out, torch.int32, "ranks_out"), self._ptr(ranks2_out, torch.int32, "ranks2_out"),
            self._ptr(grad_out, torch.float32, "grad_out"), self._stream()), "estk_rank_grad_xr_adam")
        self.launches += 1

    def clamp_adam(self, grad_sum, P, theta, m, v, state, adam, grad_out=None):
        _capi.check(self.lib.estk_clamp_adam(
            self._ctx, self._ptr(grad_sum, torch.float32, "grad_sum"), int(P), grad_sum.numel(),
            self._ptr(theta, torch.float32, "theta"), self._ptr(m, torch.float32, "m"),
            self._ptr(v, torch.float32, "v"), self._ptr(state, torch.uint8, "state"), C.byref(adam),
            self._ptr(grad_out, torch.float32, "grad_out"), self._stream()), "estk_clamp_adam")
        self.launches += 1

    # ---------------------------------------------------------------- novelty
    def knn_novelty(self, bc, archive, k, novelty_out):
        count, dim = bc.shape
        _capi.check(self.lib.estk_knn_novelty(
            self._ctx, self._ptr(bc, torch.float32, "bc"), int(count),
            self._ptr(archive, torch.float32, "archive"), int(archive.shape[0]), int(dim), int(k),
            self._ptr(novelty_out, torch.float32, "novelty_out"), self._stream()), "estk_knn_novelty")
        self.launches += 2      # frob_kernel + knn_novelty_kernel
