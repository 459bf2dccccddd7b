"""TEST-ONLY: the MLP activation codes of include/estk.h (``estk_mlp_desc.activation``) and the references of the
MLP evaluate and act modes, on the forwards of ``oracle/es_oracle.py``.

A code is hidden kind | output | loss: the hidden kind in bits 0-7 (ReLU, Tanh, ELU, SiLU, LeakyReLU), the Tanh
output in bit 8, and the loss in bits 16-23 (squared error, the cross-entropy ESTK_LOSS_XENT, the classification
accuracy ESTK_LOSS_ACCURACY; ESTK_ACTIONS in the act mode).  The evaluate defines 20 codes: the five hidden kinds
with the squared error (identity or Tanh output), the cross-entropy and the accuracy (identity output).

The returns, per member, of its fp32 outputs:
    squared error   -mean((y - t)^2) in fp32 (``orc.synthetic_return``)
    cross-entropy   -(sum_b ce_b) / B, ce_b the soft-target cross-entropy of row b reduced in fp64, rounded to fp32
    accuracy        count / B in fp32, one divide; a row counts when the first index of the maximum of its logits
                    equals the first index of the maximum of its target row (a NaN counts as the maximum:
                    ``np.argmax`` and ``torch.argmax`` agree on this)."""
import numpy as np
from torch import nn

from oracle import es_oracle as orc

ACT_TANH, ACT_ELU, ACT_SILU, ACT_LEAKY_RELU = 1, 3, 4, 5    # include/estk.h ESTK_ACT_*
ACT_OUT_TANH = 1 << 8                                      # ESTK_ACT_OUT_TANH
LOSS_XENT, ACTIONS, LOSS_ACCURACY = 1 << 16, 3 << 16, 6 << 16   # ESTK_LOSS_XENT, ESTK_ACTIONS, ESTK_LOSS_ACCURACY
HIDDEN_CODES = {"relu": 0, "tanh": ACT_TANH, "elu": ACT_ELU, "silu": ACT_SILU, "leaky_relu": ACT_LEAKY_RELU}
LOSS_CODES = {"mse": 0, "xent": LOSS_XENT, "accuracy": LOSS_ACCURACY}
NEW_KINDS = ("elu", "silu", "leaky_relu")
XENT_ACTS = (LOSS_XENT, LOSS_XENT | ACT_TANH)
# the nine codes ELU, SiLU and LeakyReLU add: squared error with identity / tanh output, and the cross-entropy
NEW_ACTS = tuple(HIDDEN_CODES[k] | extra for k in NEW_KINDS for extra in (0, ACT_OUT_TANH, LOSS_XENT))
ALL_ACTS = tuple(h | extra for h in HIDDEN_CODES.values() for extra in (0, ACT_OUT_TANH, LOSS_XENT))
ACCURACY_ACTS = tuple(h | LOSS_ACCURACY for h in HIDDEN_CODES.values())
CODES = ALL_ACTS + ACCURACY_ACTS

FORWARD = {"fp32": orc.mlp_forward, "f16": orc.mlp_forward_f16, "f16_any": orc.mlp_forward_f16,
           "bf16": orc.mlp_forward_bf16, "bf16s": orc.mlp_forward_bf16}


def decode(code):
    """A defined evaluate code -> (hidden, output, loss)."""
    assert code in CODES, hex(code)
    hidden = {v: k for k, v in HIDDEN_CODES.items()}[code & 0xff]
    loss = {v: k for k, v in LOSS_CODES.items()}[code & 0xff0000]
    return hidden, ("tanh" if code & ACT_OUT_TANH else "identity"), loss


def code(hidden="relu", output="identity", loss="mse"):
    return HIDDEN_CODES[hidden] | (ACT_OUT_TANH if output == "tanh" else 0) | LOSS_CODES[loss]


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


def correct_rows(logits, target):
    """[B] bool: the first argmax of each logits row equals the first argmax of its target row."""
    return np.argmax(np.asarray(logits), axis=1) == np.argmax(np.asarray(target), axis=1)


def accuracy_return(logits, target):
    """(float32)count / (float32)B."""
    return np.float32(np.float32(correct_rows(logits, target).sum()) / np.float32(np.asarray(logits).shape[0]))


RETURNS = {"mse": orc.synthetic_return, "xent": xent_return, "accuracy": accuracy_return}


def member_return(out, target, loss="mse"):
    return RETURNS[loss](out, target)


def evaluate_population(rows, dims, obs, target, code=0, precision="fp32", bc_obs=0, bc_dim=0):
    """Per-row rollout of the synthetic agent: returns [M] and behaviour characteristics [M, bc_dim] (None
    without a bc) of the members ``rows`` [M, n] under the evaluate code, in the precision's forward."""
    hidden, output, loss = decode(code)
    rets = np.empty(rows.shape[0], dtype=np.float32)
    bcs = np.empty((rows.shape[0], bc_dim), dtype=np.float32) if bc_dim else None
    for i in range(rows.shape[0]):
        out = FORWARD[precision](rows[i], list(dims), obs, hidden, output)
        rets[i] = member_return(out, target, loss)
        if bc_dim:
            bcs[i] = orc.synthetic_bc(out, bc_obs, bc_dim)
    return rets, bcs


def act_forward(rows, dims, obs, code):
    """The act mode of estk_eval_mlp (ESTK_ACTIONS, estorch_b200/csrc/estk_eval_mlp_act.cu): rows [M, n] (each
    member's parameters), obs [M, B, in] -> outputs [M, B, out] (fp32).  Per output one fma chain from 0 in
    ascending k, + bias in fp32, the hidden activation of ``orc.HIDDEN``, tanh in fp32 for the Tanh output.  The
    fp32 fma is emulated in fp64: the product of two fp32 values is exact there, the sum is rounded to fp64 and
    then to fp32 (a double rounding that differs from one fma rounding only in rare ties)."""
    hidden = {v: k for k, v in HIDDEN_CODES.items()}[code & 0xff]
    h = np.asarray(obs, dtype=np.float32)
    n_layers = len(dims) - 1
    layers = [orc.mlp_unflatten(r, dims) for r in np.asarray(rows, dtype=np.float32)]
    for li in range(n_layers):
        W = np.stack([lay[li][0] for lay in layers])          # [M, out, in]
        b = np.stack([lay[li][1] for lay in layers])          # [M, out]
        acc = np.zeros(h.shape[:2] + (W.shape[1],), dtype=np.float32)
        for k in range(W.shape[2]):
            acc = (acc.astype(np.float64) + h[:, :, k, None].astype(np.float64) *
                   W[:, None, :, k].astype(np.float64)).astype(np.float32)
        y = (acc + b[:, None, :]).astype(np.float32)
        h = orc.HIDDEN[hidden](y).astype(np.float32) if li + 1 < n_layers else y
    return np.tanh(h).astype(np.float32) if code & ACT_OUT_TANH else h


class MLP(nn.Module):
    """Linear -> hidden -> ... -> Linear [-> Tanh], activations as registered modules; ``hidden`` may also be
    one kind per hidden layer."""
    MODULES = {"relu": nn.ReLU, "tanh": nn.Tanh, "elu": nn.ELU, "silu": nn.SiLU, "leaky_relu": nn.LeakyReLU}

    def __init__(self, dims, hidden="relu", output="identity"):
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
