"""TEST-ONLY: the oracle's MLP forwards with the activations of include/estk.h.

``oracle/es_oracle.py`` restates the ReLU policy (Linear -> ReLU -> ... -> Linear).  The
forwards here take ``hidden="relu" | "tanh"`` and ``output="identity" | "tanh"``; with the
defaults they are the oracle's arithmetic operation for operation, so they reproduce
``orc.mlp_forward`` / ``mlp_forward_f16`` / ``mlp_forward_bf16`` bit for bit.  Rounding
model of Tanh (the kernels' epilogues): tanh of the fp32 value acc + bias; a hidden tanh
is rounded once to the 16-bit operand type in the tensor-core emulations; the output tanh
stays fp32.

``ActOracleBackend`` is the CPU stand-in of ``tests/_oracle_backend.py`` with the
``act=`` keyword of ``CudaBackend``'s MLP entry points."""
import numpy as np
import torch

from oracle import es_oracle as orc
from _oracle_backend import OracleBackend, _np

ACT_TANH, ACT_OUT_TANH = 1, 1 << 8          # include/estk.h ESTK_ACT_TANH / ESTK_ACT_OUT_TANH
ALL_ACTS = (0, ACT_TANH, ACT_OUT_TANH, ACT_TANH | ACT_OUT_TANH)


def kinds(act):
    """estk_mlp_desc.activation code -> (hidden, output)."""
    assert act in ALL_ACTS, act
    return ("tanh" if act & 0xff else "relu"), ("tanh" if act & ACT_OUT_TANH else "identity")


def code(hidden="relu", output="identity"):
    return (ACT_TANH if hidden == "tanh" else 0) | (ACT_OUT_TANH if output == "tanh" else 0)


def _hidden(h, hidden):
    return np.tanh(h) if hidden == "tanh" else np.maximum(h, np.float32(0.0))


def _output(h, output):
    return np.tanh(h).astype(np.float32) if output == "tanh" else h


def mlp_forward(flat, dims, obs, hidden="relu", output="identity"):
    """fp32 forward (orc.mlp_forward with the activations above)."""
    h = np.asarray(obs, dtype=np.float32)
    layers = orc.mlp_unflatten(np.asarray(flat, dtype=np.float32), dims)
    for li, (w, b) in enumerate(layers):
        h = (h @ w.T + b).astype(np.float32)
        if li + 1 < len(layers):
            h = _hidden(h, hidden)
    return _output(h, output)


def mlp_forward_bf16(flat, dims, obs, hidden="relu", output="identity"):
    """Emulation of the "bf16" / "bf16s" wgmma roundings (orc.mlp_forward_bf16)."""
    h = orc.round_bf16(np.asarray(obs, dtype=np.float32))
    layers = orc.mlp_unflatten(np.asarray(flat, dtype=np.float32), dims)
    for li, (w, b) in enumerate(layers):
        z = (h.astype(np.float64) @ orc.round_bf16(w).astype(np.float64).T).astype(np.float32) + b
        if li + 1 < len(layers):
            h = orc.round_bf16(_hidden(z, hidden))
        else:
            h = z.astype(np.float32)
    return _output(h, output)


def mlp_forward_f16(flat, dims, obs, hidden="relu", output="identity"):
    """Emulation of the "f16" wgmma roundings (orc.mlp_forward_f16); tanh(z) is rounded to fp16 once."""
    x = np.asarray(obs, dtype=np.float32)
    x_hi = orc.round_f16(x)
    h = x_hi.astype(np.float64) + orc.round_f16(x - x_hi).astype(np.float64)
    layers = orc.mlp_unflatten(np.asarray(flat, dtype=np.float32), dims)
    for i, (w, b) in enumerate(layers):
        h = (h @ orc.round_f16(w).astype(np.float64).T + b.astype(np.float64)).astype(np.float32)
        if i + 1 < len(layers):
            h = orc.round_f16(_hidden(h, hidden)).astype(np.float64)
    return _output(h.astype(np.float32), output)


FORWARD = {"fp32": mlp_forward, "f16": mlp_forward_f16, "bf16": mlp_forward_bf16, "bf16s": mlp_forward_bf16}


def evaluate_population(pop, dims, obs, target, bc_obs=0, bc_dim=0, hidden="relu", output="identity",
                        precision="fp32"):
    """Per-row rollout of the synthetic agent (orc.evaluate_population)."""
    fwd = FORWARD[precision]
    rets = np.empty(pop.shape[0], dtype=np.float32)
    bcs = np.empty((pop.shape[0], bc_dim), dtype=np.float32) if bc_dim else None
    for i in range(pop.shape[0]):
        out = fwd(pop[i], dims, obs, hidden, output)
        rets[i] = orc.synthetic_return(out, target)
        if bc_dim:
            bcs[i] = orc.synthetic_bc(out, bc_obs, bc_dim)
    return rets, bcs


class ActOracleBackend(OracleBackend):
    """OracleBackend whose MLP evaluate honours ``act`` in every precision mode."""

    def eval_supports_bf16(self, dims, B, act=0):
        return act in ALL_ACTS and super().eval_supports_bf16(dims, B)

    def eval_supports_f16(self, dims, B, act=0):
        return act in ALL_ACTS and super().eval_supports_f16(dims, B)

    def _rows(self, theta, table, offsets, sigma, dims, precision):
        pop, _ = orc.sample_population(_np(theta), _np(table), _np(offsets), sigma)
        if precision != "bf16s":
            return pop
        return self._exact_biases(orc.sample_population_bf16s(_np(theta), _np(table), _np(offsets), sigma), pop,
                                  list(dims))

    def eval_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                 bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", centre_out=None, act=0, **extra):
        hidden, output = kinds(act)
        if precision != "fp32":
            assert self.tensor_core
            if precision == "f16":
                t16 = extra["table16"]
                assert t16.dtype == torch.float16 and np.array_equal(_np(t16).astype(np.float32), _np(table))
        else:
            assert centre_out is None
        rows = self._rows(theta, table, offsets, sigma, dims, precision)
        rets, bcs = evaluate_population(rows, list(dims), _np(obs), _np(target), bc_obs, bc_dim, hidden, output,
                                        precision)
        ret_plus.copy_(torch.from_numpy(rets[:pairs]))
        ret_minus.copy_(torch.from_numpy(rets[pairs:]))
        if bc_plus is not None:
            bc_plus.copy_(torch.from_numpy(bcs[:pairs]))
            bc_minus.copy_(torch.from_numpy(bcs[pairs:]))
        if centre_out is not None:       # the folded post-update rollout of the previous generation
            self.centre_folds += 1
            self.eval_mlp_center(dims, theta, obs, target, centre_out, precision=precision, act=act)

    def eval_mlp_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0, precision="fp32",
                        act=0, **_):
        hidden, output = kinds(act)
        th = _np(theta)
        if precision == "bf16s":
            th = self._exact_biases(orc.round_bf16(th).copy(), th, list(dims))
        out = FORWARD[precision](th, list(dims), _np(obs), hidden, output)
        ret_out[0] = float(orc.synthetic_return(out, _np(target)))
        if bc_out is not None:
            bc_out.copy_(torch.from_numpy(orc.synthetic_bc(out, bc_obs, bc_dim)))
