"""TEST-ONLY: a float64 reference of an evaluate call, and what ES consumes of its returns.

ES does not use the returns themselves but their order: centred ranks, then the gradient
``sum_j (c+_j - c-_j) eps_j``.  The order is set by the antithetic differences ``D_j = R+_j - R-_j``,
which are O(sigma) of R -- so an evaluate can match fp32 returns to 1e-5 and still reorder members
whose differences are small.  This module states the fp64 truth of an evaluate call and measures a
return vector against it on the quantities the update sees.

* ``members``: the rows W+- of a call, formed with the kernels' two fp32 roundings
  (eps = fp32(sigma * T), W = fp32(theta +- eps); ``perturb_rows`` bit for bit).
* ``mlp_reference``: the float64 forward and return of every member, and a bound ``tau`` of an fp32
  evaluate's error on each return, from the same forward on the squares of W and h (below).
* ``cnn_reference`` / ``seq_reference`` / ``conv_vbn_reference``: float64 returns and bounds of the
  other fp32 back ends, from the float64 forwards of ``_cnn_oracle``, ``_seq_oracle`` and ``_vbn_frames``.
* ``device_gradient``: ranks and gradient of a return vector from the device's ``rank_grad_adam``.
* ``signal_metrics``: return error, pair-difference error, wrong-sign fraction, rank displacement and
  gradient rel-L2 of any return vector against the float64 one.

The bound.  The worst-case bound of an fp32 dot product of length k, (k + 1) u |W||h| (u = 2^-24), is
some 10^4 times the error a [64, 256, 256, 32] forward actually makes, and would excuse every rank of a
64-member population.  The bound here is the probabilistic one (Higham & Mary 2019): k roundings move a
sum by at most lambda sqrt(k) u times the root sum of squares of its terms, lambda = 6, and errors
carried in from the layer below add in quadrature through W.  As variances per output, in units of u^2:

    v_{l+1} = L_act^2 ((W_l o W_l) v_l) + lambda^2 (k_l + 1) ((W_l o W_l)(h_l o h_l) + b_l o b_l) + 4 h_{l+1}^2,

the same forward run on the squares of W and h (L_act: 1 for ReLU, Tanh, ELU and LeakyReLU, 1.1 for
SiLU; the 4 h^2 is the activation's own rounding).  The return inherits e = lambda u sqrt(v) through the
loss (first order: 2 |y - t| e for the squared error, 2 sum|t| max_c e for the cross-entropy) plus the
rounding of its own sum, lambda sqrt(terms) u times the sum of its absolute terms."""
import numpy as np

from oracle import es_oracle as orc

U32 = 2.0 ** -24
# Lipschitz constants of the hidden activations (SiLU's derivative peaks at 1.0998)
LIPSCHITZ = {"relu": 1.0, "tanh": 1.0, "elu": 1.0, "silu": 1.1, "leaky_relu": 1.0}
# lambda of the probabilistic rounding-error bound: k roundings of a sum move it by at most
# lambda sqrt(k) u times the root sum of squares of its terms (Higham & Mary 2019)
LAMBDA = 6.0


def _gamma(k):
    return LAMBDA * np.sqrt(k) * U32


def members(theta, table, offsets, sigma):
    """W+- of an evaluate call, [2 * pairs, n] float32: the + members in pair order, then their mirrors."""
    pop, _ = orc.sample_population(np.asarray(theta, np.float32), np.asarray(table, np.float32),
                                   np.asarray(offsets), sigma)
    return pop


def act64(kind, z):
    """The hidden activations of include/estk.h in float64."""
    if kind == "relu":
        return np.maximum(z, 0.0)
    if kind == "tanh":
        return np.tanh(z)
    if kind == "elu":
        return np.where(z > 0, z, np.expm1(np.minimum(z, 0.0)))
    if kind == "silu":
        with np.errstate(over="ignore"):            # exp(-z) = inf for z << 0: z / inf = -0
            return z / (1.0 + np.exp(-z))
    if kind == "leaky_relu":
        return np.where(z > 0, z, 0.01 * z)
    raise ValueError(kind)


def _layers(rows, dims):
    """Per Linear, (W [M, out, in], b [M, out]) of every member, float64."""
    rows = np.asarray(rows, np.float32).astype(np.float64)
    out, i = [], 0
    for fi, fo in zip(dims[:-1], dims[1:]):
        w = rows[:, i: i + fi * fo].reshape(-1, fo, fi)
        i += fi * fo
        out.append((w, rows[:, i: i + fo]))
        i += fo
    assert i == rows.shape[1]
    return out


def mlp_reference(rows, dims, obs, target, hidden="relu", output="identity", loss="mse"):
    """(R64 [M], tau [M]): the float64 return of every member row (``rows`` [M, n], fp32 values) of the MLP
    ``dims`` on ``obs`` [B, in] / ``target`` [B, out], and the bound of an fp32 evaluate's error on
    it (module docstring).  ``output``: "identity" or "tanh"; ``loss``: "mse" (-mean((y - t)^2)) or
    "xent" (-(1/B) sum_b soft-target cross-entropy of the logits y)."""
    dims = [int(d) for d in dims]
    x = np.asarray(obs, np.float32).astype(np.float64)
    t = np.asarray(target, np.float32).astype(np.float64)
    layers = _layers(rows, dims)
    M = len(layers[0][0])
    h = np.broadcast_to(x, (M,) + x.shape)
    v = np.zeros_like(h)                  # variance bound of the error carried in h, in units of u^2
    for li, (w, b) in enumerate(layers):
        wt = np.swapaxes(w, 1, 2)
        z = h @ wt + b[:, None, :]
        v = v @ (wt * wt) + LAMBDA ** 2 * (dims[li] + 1) * ((h * h) @ (wt * wt) + (b * b)[:, None, :])
        if li + 1 < len(layers):
            h = act64(hidden, z)
            v = LIPSCHITZ[hidden] ** 2 * v + 4 * h * h
        else:
            h = z
    if output == "tanh":
        h = np.tanh(h)
        v = v + 4 * h * h
    e = LAMBDA * np.sqrt(v) * U32
    B, C = h.shape[1], h.shape[2]
    if loss == "mse":
        d = h - t[None]
        R = -(d * d).mean((1, 2))
        tau = np.sqrt(((2 * d * e) ** 2).sum((1, 2))) / (B * C) + _gamma(B * C + 2) * (d * d).mean((1, 2))
    elif loss == "xent":
        m = h.max(-1, keepdims=True)
        lse = m[..., 0] + np.log(np.exp(h - m).sum(-1))
        ce = lse * t.sum(-1)[None] - (t[None] * h).sum(-1)
        R = -ce.mean(1)
        ta = np.abs(t).sum(-1)[None]
        # the per-row terms in absolute value: lse * sum(t) and sum(t * y), each with its exp/log ulps
        terms = np.abs(lse) * ta + (np.abs(t)[None] * np.abs(h)).sum(-1)
        tau = np.sqrt(((2 * ta * e.max(-1)) ** 2).sum(1)) / B + _gamma(B + C + 8) * terms.mean(1)
    else:
        raise ValueError(loss)
    return R, tau + 2 * U32 * np.abs(R)


def mse_tau(y64, target, chain):
    """The bound of an fp32 squared-error return for a back end without a layer-by-layer bound here (recurrent,
    convolutional, VirtualBatchNorm): ``y64`` [M, ...] the float64 outputs, ``target`` [...], ``chain`` the
    longest chain of roundings behind one output (the sum of the fan-ins along the way).  Each output is taken
    to carry lambda sqrt(chain) u of rounding error times chain^(1/2) rms(y) -- the |W||h| of a sum whose terms
    cancel down to |y| exceeds it by about the square root of its length."""
    y = np.asarray(y64, np.float64)
    M = len(y)
    d = (y - np.asarray(target, np.float64)[None]).reshape(M, -1)
    e = _gamma(chain) * np.sqrt(chain) * np.sqrt((y.reshape(M, -1) ** 2).mean(1))[:, None]
    k = d.shape[1]
    tau = np.sqrt(((2 * d * e) ** 2).sum(1)) / k + _gamma(k + 2) * (d * d).mean(1)
    return -(d * d).mean(1), tau


def cnn_reference(rows, dims, code, obs, target):
    """(R64, tau) of a convolutional policy with the squared error (``_cnn_oracle``'s float64 forward)."""
    import _cnn_oracle as cnn
    shape, convs, linears = cnn.unpack(dims, (int(code) >> 24) & 0xff)
    shapes, _ = cnn.layer_shapes(shape, convs, linears)
    y = np.stack([cnn.forward(r, dims, code, obs, np.float64) for r in rows])
    return mse_tau(y, target, sum(int(np.prod(ws[1:])) for ws, _ in shapes))


def seq_reference(rows, cell, dims, obs, target, out_tanh=False):
    """(R64, tau) of a recurrent sequence evaluate with the squared error (``_seq_oracle``'s float64 forward)."""
    import _seq_oracle as seq
    din, H, _ = (int(d) for d in dims)
    T = np.asarray(obs).shape[1]
    return mse_tau(seq.seq_forward64(rows, cell, dims, obs, out_tanh), target, T * (din + H) + H)


def conv_vbn_reference(rows, n_actions, xref, obs, target):
    """(R64, tau) of the conv + VirtualBatchNorm policy, -mean((y - t)^2) (``_vbn_frames.Forward64``)."""
    import _vbn_frames as vf
    y = np.stack([vf.Forward64(r, n_actions, xref)(obs) for r in rows])
    return mse_tau(y, target, 4 * 8 * 8 + 16 * 4 * 4 + 2592 + 256)


def centred_ranks(returns):
    """ES's weights of a return vector: centred ranks in [-0.5, 0.5] (stable on ties)."""
    return orc.rank_transformation(np.asarray(returns))


def gradient64(returns, table, offsets, n):
    """The pair-difference gradient of centred ranks, float64 (``orc.calculate_grad_pairs``)."""
    return orc.calculate_grad_pairs(np.asarray(returns, np.float32), np.asarray(table, np.float32),
                                    np.asarray(offsets), n)


def device_gradient(be, returns, table, offsets, order, theta):
    """(ranks [P] int64, gradient [n] float32) of ``returns`` from the device's fused rank + gradient + Adam
    step (``be.rank_grad_adam``) on the given table and offsets: the gradient the engine would apply."""
    import torch
    from estorch_b200.backend import adam_desc, new_state
    P, n = int(returns.numel()), int(theta.numel())
    th, m, v = theta.clone(), be.zeros(n), be.zeros(n)
    ranks, grad = be.zeros(P, dtype=torch.int32), be.zeros(n)
    be.rank_grad_adam(returns, None, 1.0, 0.0, P, table, offsets, order, th, m, v, new_state(be.device),
                      adam_desc(lr=0.01), ranks, None, grad)
    return ranks.cpu().numpy().astype(np.int64), grad.cpu().numpy()


def signal_metrics(returns, r64, grad=None, grad64=None):
    """What ``returns`` [P] (+ members, then their mirrors) does to ES's signal, against the float64 returns
    ``r64``: the max-norm return error, max|D - D64| / std(D64) of the pair differences, the fraction of D
    with the wrong sign, the largest and mean rank displacement, and -- given the gradients of both -- the
    gradient rel-L2."""
    r = np.asarray(returns, np.float64)
    r64 = np.asarray(r64, np.float64)
    pairs = r.size // 2
    d, d64 = r[:pairs] - r[pairs:], r64[:pairs] - r64[pairs:]
    disp = np.abs(orc.compute_ranks(r) - orc.compute_ranks(r64))
    out = {"returns_max_rel": float(np.max(np.abs(r - r64)) / np.max(np.abs(r64))),
           "diff_max_over_std": float(np.max(np.abs(d - d64)) / max(d64.std(), 1e-300)),
           "diff_wrong_sign": float(np.mean(np.sign(d) != np.sign(d64))),
           "rank_max_disp": int(disp.max()), "rank_mean_disp": float(disp.mean())}
    if grad is not None:
        g, g64 = np.asarray(grad, np.float64), np.asarray(grad64, np.float64)
        out["grad_rel_l2"] = float(np.linalg.norm(g - g64) / np.linalg.norm(g64))
    return out


def rank_violations(returns, r64, tau):
    """Members whose rank differs from their float64 rank although no float64 neighbour lies within the error
    bounds (|R64_j - R64_k| <= tau_j + tau_k), and how many members are so pinned: (violations, pinned)."""
    r64, tau = np.asarray(r64, np.float64), np.asarray(tau, np.float64)
    close = np.abs(r64[:, None] - r64[None, :]) <= tau[:, None] + tau[None, :]
    np.fill_diagonal(close, False)
    free = ~close.any(1)
    moved = orc.compute_ranks(np.asarray(returns)) != orc.compute_ranks(r64)
    return np.flatnonzero(free & moved), int(free.sum())
