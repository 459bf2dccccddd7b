"""TEST-ONLY: the classification-accuracy return (include/estk.h ESTK_LOSS_ACCURACY) on the oracle's forwards.

``accuracy_return`` restates the header: label_b and pred_b are the first index of the maximum of the target row
and of the logits (a NaN counts as the maximum: ``np.argmax`` and ``torch.argmax`` agree on this), and the return is
count / B, one fp32 divide.  The forwards are those of ``tests/_act_ext_oracle.py`` with the identity output, exact
fp32 or the emulated roundings of the tensor-core modes ("f16" / "f16_any" via ``mlp_forward_f16``).

``AccuracyOracleBackend`` is the CPU stand-in of ``tests/_act_ext_oracle.py`` that also honours the accuracy code,
under the cross-entropy's shape rules, and records every code it sees in ``acts``."""
import numpy as np
import torch

from oracle import es_oracle as orc
import _act_ext_oracle as ext
import _xent_oracle as xent
from _act_ext_oracle import ActExtOracleBackend, _np

LOSS_ACCURACY = 6 << 16                      # include/estk.h ESTK_LOSS_ACCURACY
ACCURACY_ACTS = tuple(h | LOSS_ACCURACY for h in ext.HIDDEN_CODES.values())


def is_accuracy(code):
    return (code & 0xff0000) == LOSS_ACCURACY


def correct_rows(logits, target):
    """[B] bool: the first argmax of each logits row equals the first argmax of its target row."""
    return np.argmax(np.asarray(logits), axis=1) == np.argmax(np.asarray(target), axis=1)


def accuracy_return(logits, target):
    """(float32)count / (float32)B."""
    return np.float32(np.float32(correct_rows(logits, target).sum()) / np.float32(np.asarray(logits).shape[0]))


def hidden_of(code):
    assert code in ACCURACY_ACTS, hex(code)
    return {v: k for k, v in ext.HIDDEN_CODES.items()}[code & 0xff]


def evaluate_population(pop, dims, obs, target, bc_obs=0, bc_dim=0, hidden="relu", precision="fp32"):
    fwd = ext.FORWARD[precision]
    rets = np.empty(pop.shape[0], dtype=np.float32)
    bcs = np.empty((pop.shape[0], bc_dim), dtype=np.float32) if bc_dim else None
    for i in range(pop.shape[0]):
        out = fwd(pop[i], list(dims), obs, hidden, "identity")
        rets[i] = accuracy_return(out, target)
        if bc_dim:
            bcs[i] = orc.synthetic_bc(out, bc_obs, bc_dim)
    return rets, bcs


class AccuracyOracleBackend(ActExtOracleBackend):
    """ActExtOracleBackend whose MLP evaluate also honours ESTK_LOSS_ACCURACY."""

    def eval_supports_bf16(self, dims, B, act=0):
        if is_accuracy(act):
            return act in ACCURACY_ACTS and super().eval_supports_bf16(dims, B, (act & 0xff) | xent.LOSS_XENT)
        return super().eval_supports_bf16(dims, B, act)

    def eval_supports_f16(self, dims, B, act=0):
        if is_accuracy(act):
            return act in ACCURACY_ACTS and super().eval_supports_f16(dims, B, (act & 0xff) | xent.LOSS_XENT)
        return super().eval_supports_f16(dims, B, act)

    def eval_supports_f16_any(self, dims, B, act=0):
        return self.tensor_core and B >= 1 and (act in ACCURACY_ACTS or act in ext.ALL_ACTS)

    def eval_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                 bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", centre_out=None, act=0, **extra):
        if not is_accuracy(act):
            return super().eval_mlp(dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus,
                                    ret_minus, bc_plus, bc_minus, bc_obs, bc_dim, precision, centre_out, act, **extra)
        self.acts.add(act)
        if precision != "fp32":
            assert self.tensor_core
        else:
            assert centre_out is None
        rows = self._rows(theta, table, offsets, sigma, dims, "f16" if precision == "f16_any" else precision)
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
        if not is_accuracy(act):
            return super().eval_mlp_center(dims, theta, obs, target, ret_out, bc_out, bc_obs, bc_dim, precision,
                                           act, **kw)
        self.acts.add(act)
        th = _np(theta)
        if precision == "bf16s":
            th = self._exact_biases(orc.round_bf16(th).copy(), th, list(dims))
        out = ext.FORWARD[precision](th, list(dims), _np(obs), hidden_of(act), "identity")
        ret_out[0] = float(accuracy_return(out, _np(target)))
        if bc_out is not None:
            bc_out.copy_(torch.from_numpy(orc.synthetic_bc(out, bc_obs, bc_dim)))
