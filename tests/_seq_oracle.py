"""TEST-ONLY: the recurrent sequence evaluate (estk_eval_mlp with ESTK_CELL_GRU / ESTK_CELL_LSTM and a return,
include/estk.h) in numpy -- T chained ``_rnn_oracle.step32`` steps, the fp32 restatement of the documented loss
reduction and a float64 forward --, and the supervised delayed-recall dataset of the sequence tests and goldens."""
import numpy as np
import torch

from _rnn_oracle import forward64, state_width, step32

LOSS_XENT = 1 << 16          # include/estk.h ESTK_LOSS_XENT


def _f32(a):
    return np.asarray(a, dtype=np.float32)


def _fma32(a, b, c):
    return (_f32(a).astype(np.float64) * _f32(b).astype(np.float64) + _f32(c).astype(np.float64)).astype(np.float32)


def seq_outputs32(rows, cell, dims, obs, out_tanh):
    """rows [M, n], obs [B, T, in] -> y [M, B, T, out]: T chained fp32 steps from the zero state."""
    M, (B, T, _) = len(rows), obs.shape
    S = state_width(cell, dims[1])
    state = np.zeros((M, B, S), np.float32)
    ys = []
    for t in range(T):
        x = np.broadcast_to(_f32(obs)[None, :, t], (M, B, dims[0]))
        o = step32(rows, cell, dims, np.concatenate([x, state], -1), out_tanh)
        ys.append(o[..., :dims[2]])
        state = o[..., dims[2]:]
    return np.stack(ys, 2)


def seq_forward64(rows, cell, dims, obs, out_tanh):
    """The float64 forward of the same sequences: rows [M, n], obs [B, T, in] -> y [M, B, T, out]."""
    M, (B, T, _) = len(rows), obs.shape
    S = state_width(cell, dims[1])
    state = np.zeros((M, B, S))
    ys = []
    for t in range(T):
        x = np.broadcast_to(np.asarray(obs, np.float64)[None, :, t], (M, B, dims[0]))
        o = forward64(rows, cell, dims, np.concatenate([x, state], -1), out_tanh)
        ys.append(o[..., :dims[2]])
        state = o[..., dims[2]:]
    return np.stack(ys, 2)


def seq_returns32(y, target, xent):
    """The fp32 restatement of estk.h's reduction on given outputs: y [M, B, T, C], target [B, T, C] -> [M].
    Per step a chain over c (the squared error's fmaf(d, d, s), or the cross-entropy's MLP formula), then the
    per-sequence sum in t order, the sum over sequences in b order, and -(S / count)."""
    y, tg = _f32(y), _f32(target)
    M, B, T, C = y.shape
    steps = np.zeros((M, B, T), np.float32)
    if xent:
        m = y.max(-1)
        se = np.zeros((M, B, T), np.float32)
        st = np.zeros((B, T), np.float32)
        sty = np.zeros((M, B, T), np.float32)
        for c in range(C):
            se = (se + np.exp((y[..., c] - m).astype(np.float32))).astype(np.float32)
            st = (st + tg[..., c]).astype(np.float32)
            sty = _fma32(tg[None, ..., c], y[..., c], sty)
        steps = _fma32((m + np.log(se)).astype(np.float32), st[None], -sty)
    else:
        for c in range(C):
            d = (y[..., c] - tg[None, ..., c]).astype(np.float32)
            steps = _fma32(d, d, steps)
    L = np.zeros((M, B), np.float32)
    for t in range(T):
        L = (L + steps[..., t]).astype(np.float32)
    S = np.zeros(M, np.float32)
    for b in range(B):
        S = (S + L[:, b]).astype(np.float32)
    count = np.float32(B * T * (1 if xent else C))
    return (-(S / count)).astype(np.float32)


def seq_returns64(y, target, xent):
    """The float64 return of float64 outputs y [M, B, T, C]."""
    y, tg = np.asarray(y, np.float64), np.asarray(target, np.float64)
    if xent:
        m = y.max(-1, keepdims=True)
        lsm = y - m - np.log(np.exp(y - m).sum(-1, keepdims=True))
        return (tg[None] * lsm).sum(-1).mean((1, 2))
    return -((y - tg[None]) ** 2).mean((1, 2, 3))


def recall_dataset(n_cues=3, delay=4, copies=1):
    """Supervised delayed recall: sequence b shows cue b % n_cues (one-hot) at t = 0, zeros for ``delay`` steps,
    then a recall flag at the last step (T = delay + 2).  obs [B, T, n_cues + 1]; the cross-entropy target
    [B, T, n_cues] is all zeros except the cue's one-hot at the last step, so only that step is scored.  A
    memoryless policy sees the same last observation for every cue: its best return is ``memoryless_best``."""
    K, T = n_cues, delay + 2
    B = K * copies
    obs = torch.zeros(B, T, K + 1)
    target = torch.zeros(B, T, K)
    for b in range(B):
        obs[b, 0, b % K] = 1.0
        obs[b, T - 1, K] = 1.0
        target[b, T - 1, b % K] = 1.0
    return obs, target


def memoryless_best(n_cues=3, delay=4):
    """The best return of a policy without memory on ``recall_dataset``: uniform logits at the last step,
    cross-entropy log(n_cues) per sequence, over B*T scored steps."""
    return -float(np.log(n_cues)) / (delay + 2)
