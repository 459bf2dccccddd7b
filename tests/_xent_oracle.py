"""TEST-ONLY: the cross-entropy return (include/estk.h ESTK_LOSS_XENT) on the oracle's forwards.

``xent_return`` reduces fp32 logits in fp64: the reference every kernel is measured against.  The
forwards are those of ``tests/_act_oracle.py`` with the identity output (the softmax is the output
map): exact fp32, and the emulated roundings of the "f16", "bf16" and "bf16s" tensor-core modes.

``XentOracleBackend`` is the CPU stand-in of ``tests/_act_oracle.py`` that also honours the loss
bit of ``act``."""
import numpy as np
import torch
from torch import nn

from oracle import es_oracle as orc
import _act_oracle as act
from _act_oracle import ActOracleBackend, _np

LOSS_XENT = 1 << 16                          # include/estk.h ESTK_LOSS_XENT
XENT_ACTS = (LOSS_XENT, LOSS_XENT | act.ACT_TANH)


def xent_rows(logits, target):
    """Per-row soft-target cross-entropy ce_b of fp32 logits, in fp64."""
    y = np.asarray(logits, dtype=np.float32).astype(np.float64)
    t = np.asarray(target, dtype=np.float32).astype(np.float64)
    m = y.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(y - m).sum(axis=1))
    return lse * t.sum(axis=1) - (t * y).sum(axis=1)


def xent_return(logits, target):
    """-(sum_b ce_b) / B, rounded to fp32."""
    return np.float32(-xent_rows(logits, target).sum() / np.asarray(logits).shape[0])


def hidden_of(code):
    assert code in XENT_ACTS, hex(code)
    return "tanh" if code & act.ACT_TANH else "relu"


def forward(flat, dims, obs, hidden="relu", precision="fp32"):
    return act.FORWARD[precision](flat, list(dims), obs, hidden, "identity")


def evaluate_population(pop, dims, obs, target, bc_obs=0, bc_dim=0, hidden="relu", precision="fp32"):
    rets = np.empty(pop.shape[0], dtype=np.float32)
    bcs = np.empty((pop.shape[0], bc_dim), dtype=np.float32) if bc_dim else None
    for i in range(pop.shape[0]):
        out = forward(pop[i], dims, obs, hidden, precision)
        rets[i] = xent_return(out, target)
        if bc_dim:
            bcs[i] = orc.synthetic_bc(out, bc_obs, bc_dim)
    return rets, bcs


class MLP(nn.Module):
    """Linear -> ReLU / Tanh -> ... -> Linear [-> Tanh]."""
    def __init__(self, dims, hidden="relu", output="identity"):
        super().__init__()
        layers = []
        for i in range(len(dims) - 1):
            layers.append(nn.Linear(dims[i], dims[i + 1]))
            if i + 2 < len(dims):
                layers.append(nn.Tanh() if hidden == "tanh" else nn.ReLU())
        if output == "tanh":
            layers.append(nn.Tanh())
        self.net = nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


class XentOracleBackend(ActOracleBackend):
    """ActOracleBackend whose MLP evaluate also honours ESTK_LOSS_XENT; records every code it sees."""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.acts = set()

    def eval_supports_bf16(self, dims, B, act=0):
        if act & LOSS_XENT:
            return act in XENT_ACTS and super().eval_supports_bf16(dims, B, act & ~LOSS_XENT)
        return super().eval_supports_bf16(dims, B, act)

    def eval_supports_f16(self, dims, B, act=0):
        if act & LOSS_XENT:
            return act in XENT_ACTS and super().eval_supports_f16(dims, B, act & ~LOSS_XENT)
        return super().eval_supports_f16(dims, B, act)

    def eval_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                 bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", centre_out=None, act=0, **extra):
        self.acts.add(act)
        if not act & LOSS_XENT:
            return super().eval_mlp(dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus,
                                    ret_minus, bc_plus, bc_minus, bc_obs, bc_dim, precision, centre_out, act, **extra)
        if precision != "fp32":
            assert self.tensor_core
        else:
            assert centre_out is None
        rows = self._rows(theta, table, offsets, sigma, dims, precision)
        rets, bcs = evaluate_population(rows, dims, _np(obs), _np(target), bc_obs, bc_dim, hidden_of(act), precision)
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
        self.acts.add(act)
        if not act & LOSS_XENT:
            return super().eval_mlp_center(dims, theta, obs, target, ret_out, bc_out, bc_obs, bc_dim, precision,
                                           act, **kw)
        th = _np(theta)
        if precision == "bf16s":
            th = self._exact_biases(orc.round_bf16(th).copy(), th, list(dims))
        out = forward(th, dims, _np(obs), hidden_of(act), precision)
        ret_out[0] = float(xent_return(out, _np(target)))
        if bc_out is not None:
            bc_out.copy_(torch.from_numpy(orc.synthetic_bc(out, bc_obs, bc_dim)))
