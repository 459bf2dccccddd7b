"""TEST-ONLY: the oracle's MLP forwards with the ELU, SiLU and LeakyReLU hidden activations of
include/estk.h (ESTK_ACT_ELU / ESTK_ACT_SILU / ESTK_ACT_LEAKY_RELU).

The forwards are those of ``tests/_act_oracle.py`` -- the same operations and roundings -- with the
hidden activation taken from ``HIDDEN``; for ``"relu"`` / ``"tanh"`` they call that module's own.
Rounding model of the new kinds (the kernels' epilogues): the activation of the fp32 value
y = acc + bias in fp32,

    elu         y > 0 ? y : expm1(y)
    silu        y / (1 + exp(-y))          (one fp32 divide)
    leaky_relu  y > 0 ? y : y * 0.01

then, in the tensor-core emulations, one rounding to the 16-bit operand type (fp16 saturating at
+-65504).  The output activation (identity / tanh) and the losses are unchanged.

``ActExtOracleBackend`` is the CPU stand-in of ``tests/_xent_oracle.py`` that accepts every defined
activation code: the 15 of estk.h."""
import numpy as np
import torch
from torch import nn

from oracle import es_oracle as orc
import _act_oracle as act
import _xent_oracle as xent
from _xent_oracle import XentOracleBackend, _np

ACT_ELU, ACT_SILU, ACT_LEAKY_RELU = 3, 4, 5      # include/estk.h
HIDDEN_CODES = {"relu": 0, "tanh": act.ACT_TANH, "elu": ACT_ELU, "silu": ACT_SILU, "leaky_relu": ACT_LEAKY_RELU}
NEW_KINDS = ("elu", "silu", "leaky_relu")
# the nine codes the new kinds add: squared error with identity / tanh output, and the cross-entropy
NEW_ACTS = tuple(HIDDEN_CODES[k] | extra for k in NEW_KINDS for extra in (0, act.ACT_OUT_TANH, xent.LOSS_XENT))
ALL_ACTS = tuple(h | extra for h in HIDDEN_CODES.values() for extra in (0, act.ACT_OUT_TANH, xent.LOSS_XENT))


def _elu(h):
    with np.errstate(over="ignore"):
        return np.where(h > 0, h, np.expm1(h)).astype(np.float32)


def _silu(h):
    with np.errstate(over="ignore"):
        return (h / (np.float32(1.0) + np.exp(-h))).astype(np.float32)


def _leaky_relu(h):
    return np.where(h > 0, h, h * np.float32(0.01)).astype(np.float32)


HIDDEN = {"relu": lambda h: np.maximum(h, np.float32(0.0)), "tanh": np.tanh, "elu": _elu, "silu": _silu,
          "leaky_relu": _leaky_relu}


def decode(code):
    """estk_mlp_desc.activation -> (hidden, output, loss)."""
    assert code in ALL_ACTS, hex(code)
    hidden = {v: k for k, v in HIDDEN_CODES.items()}[code & 0xff]
    return hidden, ("tanh" if code & act.ACT_OUT_TANH else "identity"), ("xent" if code & xent.LOSS_XENT else "mse")


def code(hidden="relu", output="identity", loss="mse"):
    return HIDDEN_CODES[hidden] | (act.ACT_OUT_TANH if output == "tanh" else 0) | (xent.LOSS_XENT if loss == "xent" else 0)


def mlp_forward(flat, dims, obs, hidden="relu", output="identity"):
    """fp32 forward."""
    if hidden in ("relu", "tanh"):
        return act.mlp_forward(flat, dims, obs, hidden, output)
    h = np.asarray(obs, dtype=np.float32)
    layers = orc.mlp_unflatten(np.asarray(flat, dtype=np.float32), dims)
    for li, (w, b) in enumerate(layers):
        h = (h @ w.T + b).astype(np.float32)
        if li + 1 < len(layers):
            h = HIDDEN[hidden](h)
    return act._output(h, output)


def mlp_forward_bf16(flat, dims, obs, hidden="relu", output="identity"):
    """Emulation of the "bf16" / "bf16s" wgmma roundings."""
    if hidden in ("relu", "tanh"):
        return act.mlp_forward_bf16(flat, dims, obs, hidden, output)
    h = orc.round_bf16(np.asarray(obs, dtype=np.float32))
    layers = orc.mlp_unflatten(np.asarray(flat, dtype=np.float32), dims)
    for li, (w, b) in enumerate(layers):
        z = (h.astype(np.float64) @ orc.round_bf16(w).astype(np.float64).T).astype(np.float32) + b
        if li + 1 < len(layers):
            h = orc.round_bf16(HIDDEN[hidden](z))
        else:
            h = z.astype(np.float32)
    return act._output(h, output)


def mlp_forward_f16(flat, dims, obs, hidden="relu", output="identity"):
    """Emulation of the "f16" / "f16_any" wgmma roundings: the fp32 activation rounded to fp16 once."""
    if hidden in ("relu", "tanh"):
        return act.mlp_forward_f16(flat, dims, obs, hidden, output)
    x = np.asarray(obs, dtype=np.float32)
    x_hi = orc.round_f16(x)
    h = x_hi.astype(np.float64) + orc.round_f16(x - x_hi).astype(np.float64)
    layers = orc.mlp_unflatten(np.asarray(flat, dtype=np.float32), dims)
    for i, (w, b) in enumerate(layers):
        h = (h @ orc.round_f16(w).astype(np.float64).T + b.astype(np.float64)).astype(np.float32)
        if i + 1 < len(layers):
            h = orc.round_f16(HIDDEN[hidden](h)).astype(np.float64)
    return act._output(h.astype(np.float32), output)


FORWARD = {"fp32": mlp_forward, "f16": mlp_forward_f16, "f16_any": mlp_forward_f16, "bf16": mlp_forward_bf16,
           "bf16s": mlp_forward_bf16}


def member_return(out, target, loss="mse"):
    return xent.xent_return(out, target) if loss == "xent" else orc.synthetic_return(out, target)


def evaluate_population(pop, dims, obs, target, bc_obs=0, bc_dim=0, hidden="relu", output="identity",
                        precision="fp32", loss="mse"):
    """Per-row rollout of the synthetic agent (squared error or cross-entropy)."""
    fwd = FORWARD[precision]
    rets = np.empty(pop.shape[0], dtype=np.float32)
    bcs = np.empty((pop.shape[0], bc_dim), dtype=np.float32) if bc_dim else None
    for i in range(pop.shape[0]):
        out = fwd(pop[i], list(dims), obs, hidden, output)
        rets[i] = member_return(out, target, loss)
        if bc_dim:
            bcs[i] = orc.synthetic_bc(out, bc_obs, bc_dim)
    return rets, bcs


class MLP(nn.Module):
    """Linear -> hidden -> ... -> Linear [-> Tanh], activations as registered modules."""
    MODULES = {"relu": nn.ReLU, "tanh": nn.Tanh, "elu": nn.ELU, "silu": nn.SiLU, "leaky_relu": nn.LeakyReLU}

    def __init__(self, dims, hidden="elu", output="identity"):
        super().__init__()
        layers = []
        for i in range(len(dims) - 1):
            layers.append(nn.Linear(dims[i], dims[i + 1]))
            if i + 2 < len(dims):
                layers.append(self.MODULES[hidden[i] if isinstance(hidden, (list, tuple)) else hidden]())
        if output == "tanh":
            layers.append(nn.Tanh())
        self.net = nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


class ActExtOracleBackend(XentOracleBackend):
    """XentOracleBackend that accepts every defined activation code, the new hidden kinds included,
    in every precision mode; records every code it sees in ``acts``."""

    def eval_supports_bf16(self, dims, B, act=0):
        return act in ALL_ACTS and XentOracleBackend.eval_supports_bf16(self, dims, B, 0)

    def eval_supports_f16(self, dims, B, act=0):
        return act in ALL_ACTS and XentOracleBackend.eval_supports_f16(self, dims, B, 0)

    def eval_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                 bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", centre_out=None, act=0, **extra):
        hidden, output, loss = decode(act)
        if hidden in ("relu", "tanh"):
            return super().eval_mlp(dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus,
                                    ret_minus, bc_plus, bc_minus, bc_obs, bc_dim, precision, centre_out, act, **extra)
        self.acts.add(act)
        if precision != "fp32":
            assert self.tensor_core
        else:
            assert centre_out is None
        rows = self._rows(theta, table, offsets, sigma, dims, precision)
        rets, bcs = evaluate_population(rows, dims, _np(obs), _np(target), bc_obs, bc_dim, hidden, output,
                                        precision, loss)
        ret_plus.copy_(torch.from_numpy(rets[:pairs]))
        ret_minus.copy_(torch.from_numpy(rets[pairs:]))
        if bc_plus is not None:
            bc_plus.copy_(torch.from_numpy(bcs[:pairs]))
            bc_minus.copy_(torch.from_numpy(bcs[pairs:]))
        if centre_out is not None:
            self.centre_folds += 1
            self.eval_mlp_center(dims, theta, obs, target, centre_out, precision=precision, act=act)

    def eval_mlp_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0, precision="fp32",
                        act=0, **kw):
        hidden, output, loss = decode(act)
        if hidden in ("relu", "tanh"):
            return super().eval_mlp_center(dims, theta, obs, target, ret_out, bc_out, bc_obs, bc_dim, precision,
                                           act, **kw)
        self.acts.add(act)
        th = _np(theta)
        if precision == "bf16s":
            th = self._exact_biases(orc.round_bf16(th).copy(), th, list(dims))
        out = FORWARD[precision](th, list(dims), _np(obs), hidden, output)
        ret_out[0] = float(member_return(out, _np(target), loss))
        if bc_out is not None:
            bc_out.copy_(torch.from_numpy(orc.synthetic_bc(out, bc_obs, bc_dim)))
