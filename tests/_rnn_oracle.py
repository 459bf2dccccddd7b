"""TEST-ONLY: one step of estk_eval_mlp with a recurrent cell code (ESTK_CELL_GRU / ESTK_CELL_LSTM and
ESTK_ACTIONS) in numpy -- an fp32 restatement and a float64 forward --, the recurrent policy module, and a
deterministic recall task for the population-mode tests and goldens.

Rounding model of the kernel (estorch_b200/csrc/estk_act_rnn.cu, stated in include/estk.h):
W = theta +- (sigma*t) with two fp32 roundings; per gate row two fma chains from 0 in ascending k (x against
weight_ih, h against weight_hh), each + its own bias; s(v) = 1/(1 + exp(-v)); GRU n = tanh(fma(r, b_n, a_n)),
h' = fma(z, h - n, n); LSTM c' = fma(f, c, i*g), h' = o*tanh(c'); the head is one fma chain + bias [+ tanh].
The fp32 fma is emulated in fp64 (the product of two fp32 values is exact there; the sum is rounded to fp64,
then to fp32), and exp / tanh are numpy's fp32 functions, so the restatement agrees with the kernel to a few
ulp per operation rather than bit for bit."""
import numpy as np
import torch

from estorch_b200 import PopulationAgent

ACTIONS = 3 << 16            # include/estk.h ESTK_ACTIONS
OUT_TANH = 1 << 8
CELL_GRU, CELL_LSTM = 8, 9   # include/estk.h ESTK_CELL_GRU / ESTK_CELL_LSTM
CELLS = {"gru": CELL_GRU, "lstm": CELL_LSTM}


def gates(cell):
    return 3 if cell == "gru" else 4


def state_width(cell, H):
    return H if cell == "gru" else 2 * H


def param_count(cell, dims):
    i, h, o = dims
    return gates(cell) * h * (i + h + 2) + o * (h + 1)


def unflatten(row, cell, dims):
    """A flat parameter row -> (w_ih [GH, in], w_hh [GH, H], b_ih, b_hh, w_head [out, H], b_head), torch's order."""
    i, h, o = dims
    GH = gates(cell) * h
    sizes = [GH * i, GH * h, GH, GH, o * h, o]
    shapes = [(GH, i), (GH, h), (GH,), (GH,), (o, h), (o,)]
    parts, at = [], 0
    for n, s in zip(sizes, shapes):
        parts.append(np.asarray(row[at:at + n]).reshape(s))
        at += n
    assert at == len(row)
    return parts


def policy_class(cell, out_tanh=False):
    """The recurrent policy convention: one GRUCell / LSTMCell, one Linear head, optionally a Tanh output.
    ``forward(x, state=None) -> (y, new_state)``; x and the state may carry any leading dimensions."""
    cell_t = torch.nn.GRUCell if cell == "gru" else torch.nn.LSTMCell

    class RecurrentPolicy(torch.nn.Module):
        def __init__(self, dims):
            super().__init__()
            self.cell = cell_t(dims[0], dims[1])
            self.head = torch.nn.Linear(dims[1], dims[2])
            if out_tanh:
                self.out = torch.nn.Tanh()

        def forward(self, x, state=None):
            lead = x.shape[:-1]
            flat = lambda t: t.reshape(-1, t.shape[-1])       # noqa: E731
            back = lambda t: t.reshape(*lead, t.shape[-1])    # noqa: E731
            if state is not None:
                state = flat(state) if cell == "gru" else tuple(flat(s) for s in state)
            s = self.cell(flat(x), state)
            h = s if cell == "gru" else s[0]
            y = self.head(h)
            y = back(self.out(y) if out_tanh else y)
            return y, (back(s) if cell == "gru" else tuple(back(t) for t in s))
    RecurrentPolicy.__name__ = f"{cell.upper()}Policy"
    return RecurrentPolicy


def _f32(a):
    return np.asarray(a, dtype=np.float32)


def _fma32(a, b, c):
    return (_f32(a).astype(np.float64) * _f32(b).astype(np.float64) + _f32(c).astype(np.float64)).astype(np.float32)


def _chain32(x, W):
    """x [M, B, K], W [M, N, K] -> [M, B, N]: per (row, output) one fma chain from 0 in ascending k."""
    acc = np.zeros(x.shape[:2] + (W.shape[1],), dtype=np.float32)
    for k in range(W.shape[2]):
        acc = _fma32(x[:, :, k, None], W[:, None, :, k], acc)
    return acc


def _sig32(v):
    one = np.float32(1)
    return (one / (one + np.exp(-_f32(v)))).astype(np.float32)


def step32(rows, cell, dims, xs, out_tanh):
    """The fp32 restatement: rows [M, n], xs [M, B, in + S] -> [M, B, out + S]."""
    i, H, o = dims
    xs = _f32(xs)
    parts = [unflatten(r, cell, dims) for r in _f32(rows)]
    W = [np.stack([p[k] for p in parts]) for k in range(6)]
    x, h = xs[..., :i], xs[..., i:i + H]
    a = _chain32(x, W[0]) + W[2][:, None, :]
    b = _chain32(h, W[1]) + W[3][:, None, :]
    a, b = a.astype(np.float32), b.astype(np.float32)
    g = lambda t, k: t[..., k * H:(k + 1) * H]     # noqa: E731
    if cell == "gru":
        r, z = _sig32(g(a, 0) + g(b, 0)), _sig32(g(a, 1) + g(b, 1))
        n = np.tanh(_fma32(r, g(b, 2), g(a, 2))).astype(np.float32)
        hn = _fma32(z, (h - n).astype(np.float32), n)
        state = [hn]
    else:
        c = xs[..., i + H:i + 2 * H]
        pre = (a + b).astype(np.float32)
        ig, fg, og = _sig32(g(pre, 0)), _sig32(g(pre, 1)), _sig32(g(pre, 3))
        gg = np.tanh(g(pre, 2)).astype(np.float32)
        cn = _fma32(fg, c, (ig * gg).astype(np.float32))
        hn = (og * np.tanh(cn)).astype(np.float32)
        state = [hn, cn]
    y = (_chain32(hn, W[4]) + W[5][:, None, :]).astype(np.float32)
    if out_tanh:
        y = np.tanh(y).astype(np.float32)
    return np.concatenate([y] + state, -1)


def forward64(rows, cell, dims, xs, out_tanh):
    """The float64 forward of the same step (the fp32 parameters and inputs, exactly, computed in fp64)."""
    i, H, o = dims
    xs = np.asarray(xs, dtype=np.float64)
    parts = [unflatten(np.asarray(r, dtype=np.float64), cell, dims) for r in np.asarray(rows, dtype=np.float32)]
    W = [np.stack([p[k] for p in parts]) for k in range(6)]
    x, h = xs[..., :i], xs[..., i:i + H]
    a = np.einsum("mbk,mnk->mbn", x, W[0]) + W[2][:, None, :]
    b = np.einsum("mbk,mnk->mbn", h, W[1]) + W[3][:, None, :]
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))      # noqa: E731
    g = lambda t, k: t[..., k * H:(k + 1) * H]     # noqa: E731
    if cell == "gru":
        r, z = sig(g(a, 0) + g(b, 0)), sig(g(a, 1) + g(b, 1))
        n = np.tanh(g(a, 2) + r * g(b, 2))
        hn = (1 - z) * n + z * h
        state = [hn]
    else:
        c = xs[..., i + H:i + 2 * H]
        pre = a + b
        cn = sig(g(pre, 1)) * c + sig(g(pre, 0)) * np.tanh(g(pre, 2))
        hn = sig(g(pre, 3)) * np.tanh(cn)
        state = [hn, cn]
    y = np.einsum("mbk,mnk->mbn", hn, W[4]) + W[5][:, None, :]
    if out_tanh:
        y = np.tanh(y)
    return np.concatenate([y] + state, -1)


def cell_of(code):
    return {CELL_GRU: "gru", CELL_LSTM: "lstm"}[code & 0xff]


class RecallAgent(PopulationAgent):
    """A cue-recall task: at t = 0 the observation shows one of ``n_cues`` cues (one-hot), then ``delay``
    blank steps follow, and at the last step a recall flag is shown and the policy must output the cue's
    target (0.8 at the cue's index, -0.8 elsewhere).  Every member runs all cues side by side (the batch
    dimension B = n_cues), so the return -- minus the mean squared error of the last step's outputs over
    the cues -- is deterministic.  A memoryless policy sees the same last observation for every cue and
    cannot do better than ``MEMORYLESS_BEST``.  ``bc_dim`` > 0 (= n_cues * n_cues) makes it an NS-family
    agent: the behaviour characteristic is the last step's outputs."""

    MEMORYLESS_BEST = -0.56889

    def __init__(self, delay=3, n_cues=3, bc_dim=0):
        self.delay, self.n_cues, self.bc_dim = int(delay), int(n_cues), int(bc_dim)
        assert bc_dim in (0, n_cues * n_cues)

    @property
    def obs_dim(self):
        return self.n_cues + 1

    def rollout_population(self, act, members):
        dev, K = self.device, self.n_cues
        eye = torch.eye(K, device=dev)
        first = torch.zeros(members, K, K + 1, device=dev)
        first[:, :, :K] = eye
        blank = torch.zeros(members, K, K + 1, device=dev)
        last = blank.clone()
        last[:, :, K] = 1.0
        target = 1.6 * eye - 0.8
        state = None
        for t in range(self.delay + 2):
            obs = first if t == 0 else last if t == self.delay + 1 else blank
            y, state = act(obs, state)
        ret = -((y - target) ** 2).mean((1, 2))
        if self.bc_dim:
            return ret, y.reshape(members, -1)
        return ret
