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


def mlp_desc(dims: Sequence[int], act: int = 0) -> _capi.EstkMlpDesc:
    """``act``: the ``estk_mlp_desc.activation`` code (``MLPSpec.act``; 0 = ReLU hidden, identity output)."""
    if not (2 <= len(dims) <= _capi.ESTK_MAX_LAYERS + 1):
        raise ValueError(f"MLP with {len(dims) - 1} Linear layers is outside 1..{_capi.ESTK_MAX_LAYERS}")
    d = _capi.EstkMlpDesc()
    d.n_layers = len(dims) - 1
    for i, w in enumerate(dims):
        d.dims[i] = int(w)
    d.activation = int(act)
    return d


def adam_desc(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, clamp=1.0) -> _capi.EstkAdamDesc:
    a = _capi.EstkAdamDesc()
    a.lr, a.beta1, a.beta2, a.eps = float(lr), float(betas[0]), float(betas[1]), float(eps)
    a.weight_decay, a.clamp = float(weight_decay), float(clamp)
    return a


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
        if t is None:
            return None
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

    # ---------------------------------------------------------------- evaluate
    def eval_supports_bf16(self, dims, B, act=0) -> bool:
        d = mlp_desc(dims, act)
        return bool(self.lib.estk_eval_mlp_bf16_supported(C.byref(d), int(B)))

    def eval_supports_f16(self, dims, B, act=0) -> bool:
        d = mlp_desc(dims, act)
        return bool(self.lib.estk_eval_mlp_f16_supported(C.byref(d), int(B)))

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

    def eval_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, target,
                 ret_plus, ret_minus, bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32",
                 theta16=None, table16=None, centre_out=None, act=0):
        d = mlp_desc(dims, act)
        if obs.shape != (obs.shape[0], dims[0]) or target.shape != (obs.shape[0], dims[-1]):
            raise ValueError(f"obs {tuple(obs.shape)} / target {tuple(target.shape)} do not match dims {list(dims)}")
        common = (self._ptr(offsets, torch.int64, "offsets"), self._ptr(order, torch.int32, "order"), int(pairs),
                  float(sigma), self._ptr(obs, torch.float32, "obs"), self._ptr(target, torch.float32, "target"),
                  int(obs.shape[0]), self._ptr(ret_plus, torch.float32, "ret_plus"),
                  self._ptr(ret_minus, torch.float32, "ret_minus"), self._ptr(bc_plus, torch.float32, "bc_plus"),
                  self._ptr(bc_minus, torch.float32, "bc_minus"), int(bc_obs), int(bc_dim))
        stream = (self._stream(),)
        if precision in ("f16", "bf16", "bf16s"):
            stream = (self._ptr(centre_out, torch.float32, "centre_out"), self._stream())
        elif centre_out is not None:
            raise ValueError("centre_out (folded post-update rollout) needs a tensor-core precision mode")
        common = common + stream
        th, tb = self._ptr(theta, torch.float32, "theta"), self._ptr(table, torch.float32, "table")
        if precision == "f16":
            if table16 is None:
                raise ValueError("precision='f16' needs table16, the exact fp16 copy of the table (see shadow_f16)")
            rc = self.lib.estk_eval_mlp_f16(self._ctx, C.byref(d), th, tb,
                                            self._ptr(table16, torch.float16, "table16"), *common)
        elif precision == "bf16s":
            if theta16 is None or table16 is None:
                raise ValueError("precision='bf16s' needs theta16 and table16 (see shadow_bf16)")
            rc = self.lib.estk_eval_mlp_bf16s(self._ctx, C.byref(d), th, self._ptr(theta16, torch.bfloat16, "theta16"),
                                              tb, self._ptr(table16, torch.bfloat16, "table16"), *common)
        elif precision == "bf16":
            rc = self.lib.estk_eval_mlp_bf16(self._ctx, C.byref(d), th, tb, *common)
        elif precision == "fp32":
            rc = self.lib.estk_eval_mlp(self._ctx, C.byref(d), th, tb, *common)
        else:
            raise ValueError(f"unknown precision {precision!r}")
        _capi.check(rc, "estk_eval_mlp[" + precision + "]")
        self.launches += 2 if precision == "f16" else 1      # f16: observation image + evaluate

    def eval_mlp_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0,
                        precision="fp32", theta16=None, act=0):
        d = mlp_desc(dims, act)
        tail = (self._ptr(obs, torch.float32, "obs"), self._ptr(target, torch.float32, "target"),
                int(obs.shape[0]), self._ptr(ret_out, torch.float32, "ret_out"),
                self._ptr(bc_out, torch.float32, "bc_out"), int(bc_obs), int(bc_dim), self._stream())
        th = self._ptr(theta, torch.float32, "theta")
        if precision == "f16":
            rc = self.lib.estk_eval_mlp_center_f16(self._ctx, C.byref(d), th, *tail)
        elif precision == "bf16s":
            rc = self.lib.estk_eval_mlp_center_bf16s(self._ctx, C.byref(d), th,
                                                     self._ptr(theta16, torch.bfloat16, "theta16"), *tail)
        elif precision == "bf16":
            rc = self.lib.estk_eval_mlp_center_bf16(self._ctx, C.byref(d), th, *tail)
        else:
            rc = self.lib.estk_eval_mlp_center(self._ctx, C.byref(d), th, *tail)
        _capi.check(rc, "estk_eval_mlp_center[" + precision + "]")
        self.launches += 2 if precision == "f16" else 1

    def conv_scratch_bytes(self, ref_batch, B, precision="fp32") -> int:
        if precision == "f16":
            return int(self.lib.estk_eval_conv_vbn_f16_scratch_bytes(self._ctx, int(ref_batch), int(B)))
        if precision != "fp32":
            raise ValueError(f"the conv + VirtualBatchNorm evaluate has no {precision!r} mode")
        return int(self.lib.estk_eval_conv_vbn_scratch_bytes(self._ctx, int(ref_batch), int(B)))

    def eval_conv_vbn(self, n_actions, theta, table, offsets, order, pairs, sigma, xref, obs, target,
                      ret_plus, ret_minus, scratch, precision="fp32", table16=None):
        """Conv + VirtualBatchNorm policy (examples/atari.py:14-37); offsets None = centre.
        precision "f16": the tensor-core kernel (needs table16 with offsets, and a scratch of
        conv_scratch_bytes(R, B, "f16") bytes)."""
        head = (self._ctx, int(n_actions), self._ptr(theta, torch.float32, "theta"),
                self._ptr(table, torch.float32, "table"))
        tail = (self._ptr(offsets, torch.int64, "offsets"),
                self._ptr(order, torch.int32, "order"), int(pairs), float(sigma),
                self._ptr(xref, torch.float32, "xref"), int(xref.shape[0]), self._ptr(obs, torch.float32, "obs"),
                self._ptr(target, torch.float32, "target"), int(obs.shape[0]),
                self._ptr(ret_plus, torch.float32, "ret_plus"), self._ptr(ret_minus, torch.float32, "ret_minus"),
                self._ptr(scratch, torch.uint8, "scratch"), scratch.numel(), self._stream())
        if precision == "f16":
            if offsets is not None and table16 is None:
                raise ValueError("precision='f16' needs table16, the exact fp16 copy of the table (see shadow_f16)")
            rc = self.lib.estk_eval_conv_vbn_f16(*head, self._ptr(table16, torch.float16, "table16"), *tail)
        elif precision == "fp32":
            rc = self.lib.estk_eval_conv_vbn(*head, *tail)
        else:
            raise ValueError(f"the conv + VirtualBatchNorm evaluate has no {precision!r} mode")
        _capi.check(rc, "estk_eval_conv_vbn[" + precision + "]")
        self.launches += 1

    def track_best(self, state, reward, theta, best_theta):
        _capi.check(self.lib.estk_track_best(
            self._ctx, self._ptr(state, torch.uint8, "state"), self._ptr(reward, torch.float32, "reward"),
            self._ptr(theta, torch.float32, "theta"), self._ptr(best_theta, torch.float32, "best_theta"),
            theta.numel(), self._stream()), "estk_track_best")
        self.launches += 1

    # ---------------------------------------------------------------- rank + grad + Adam
    def rank_grad_adam(self, returns, novelty, w_rew, w_nov, P, table, offsets, order, theta, m, v,
                       state, adam, ranks_out=None, ranks2_out=None, grad_out=None):
        """``table`` float32, or float16 = the exact 16-bit copy (half the bytes, same result)."""
        h = table.dtype == torch.float16
        fn = self.lib.estk_rank_grad_adam_h if h else self.lib.estk_rank_grad_adam
        _capi.check(fn(
            self._ctx, self._ptr(returns, torch.float32, "returns"),
            self._ptr(novelty, torch.float32, "novelty"), float(w_rew), float(w_nov), int(P),
            self._ptr(table, table.dtype if h else torch.float32, "table"), self._ptr(offsets, torch.int64, "offsets"),
            self._ptr(order, torch.int32, "order"), theta.numel(),
            self._ptr(theta, torch.float32, "theta"), self._ptr(m, torch.float32, "m"),
            self._ptr(v, torch.float32, "v"), self._ptr(state, torch.uint8, "state"), C.byref(adam),
            self._ptr(ranks_out, torch.int32, "ranks_out"), self._ptr(ranks2_out, torch.int32, "ranks2_out"),
            self._ptr(grad_out, torch.float32, "grad_out"), self._stream()), "estk_rank_grad_adam")
        self.launches += 1

    def rank_grad(self, returns, novelty, w_rew, w_nov, P, table, offsets, order, pair_begin,
                  pairs_local, n, grad_sum_out, ranks_out=None, ranks2_out=None, world=1):
        """``table`` float32 (member-order returns only), or float16 = the exact 16-bit copy;
        with the latter ``world > 1`` declares rank-major returns ``[world][2][pairs/world]``."""
        tail = (self._ptr(offsets, torch.int64, "offsets"),
                self._ptr(order, torch.int32, "order"), int(pair_begin), int(pairs_local), int(n),
                self._ptr(grad_sum_out, torch.float32, "grad_sum_out"),
                self._ptr(ranks_out, torch.int32, "ranks_out"), self._ptr(ranks2_out, torch.int32, "ranks2_out"),
                self._stream())
        head = (self._ctx, self._ptr(returns, torch.float32, "returns"),
                self._ptr(novelty, torch.float32, "novelty"), float(w_rew), float(w_nov), int(P))
        if table.dtype == torch.float16:
            rc = self.lib.estk_rank_grad_h(*head, int(world), self._ptr(table, torch.float16, "table16"), *tail)
        else:
            if world != 1:
                raise ValueError("rank-major returns (world > 1) need the fp16 table entry point")
            rc = self.lib.estk_rank_grad(*head, self._ptr(table, torch.float32, "table"), *tail)
        _capi.check(rc, "estk_rank_grad")
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
        _capi.check(self.lib.estk_rank_grad_xr_adam_h(
            self._ctx, self._ptr(returns, torch.float32, "returns"), self._ptr(novelty, torch.float32, "novelty"),
            float(w_rew), float(w_nov), int(P), int(world), int(rank), self._ptr(table16, torch.float16, "table16"),
            self._ptr(offsets, torch.int64, "offsets"), self._ptr(order, torch.int32, "order"), int(pair_begin),
            int(pairs_local), theta.numel(), arr, self._ptr(theta, torch.float32, "theta"),
            self._ptr(m, torch.float32, "m"), self._ptr(v, torch.float32, "v"), self._ptr(state, torch.uint8, "state"),
            C.byref(adam), self._ptr(ranks_out, torch.int32, "ranks_out"), self._ptr(ranks2_out, torch.int32, "ranks2_out"),
            self._ptr(grad_out, torch.float32, "grad_out"), self._stream()), "estk_rank_grad_xr_adam_h")
        self.launches += 1

    def clamp_adam(self, grad_sum, P, theta, m, v, state, adam, grad_out=None):
        _capi.check(self.lib.estk_clamp_adam(
            self._ctx, self._ptr(grad_sum, torch.float32, "grad_sum"), int(P), grad_sum.numel(),
            self._ptr(theta, torch.float32, "theta"), self._ptr(m, torch.float32, "m"),
            self._ptr(v, torch.float32, "v"), self._ptr(state, torch.uint8, "state"), C.byref(adam),
            self._ptr(grad_out, torch.float32, "grad_out"), self._stream()), "estk_clamp_adam")
        self.launches += 2 if theta is not None else 1

    # ---------------------------------------------------------------- novelty
    def knn_novelty(self, bc, archive, k, novelty_out):
        count, dim = bc.shape
        _capi.check(self.lib.estk_knn_novelty(
            self._ctx, self._ptr(bc, torch.float32, "bc"), int(count),
            self._ptr(archive, torch.float32, "archive"), int(archive.shape[0]), int(dim), int(k),
            self._ptr(novelty_out, torch.float32, "novelty_out"), self._stream()), "estk_knn_novelty")
        self.launches += 2
