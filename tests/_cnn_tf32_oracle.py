"""TEST-ONLY: the TF32 convolutional evaluate (include/estk_eval_cnn_tf32.h) restated in numpy -- ``rna_tf32``
(round to nearest, ties away from zero, to an 11-bit significand), the forward of a member's formed fp32 weights
with every weight and every layer input rounded that way and float64 sums -- and a stand-in backend that serves
``precision="tf32"`` with it, so the engine's mode selection runs without a GPU."""
import numpy as np
import torch

from oracle import es_oracle as orc
from _cnn_oracle import HIDDEN, LOSS_XENT, CnnOracleBackend, _act, layer_shapes, unpack
from _oracle_backend import _np

LOSS_ACCURACY = 6 << 16


def rna_tf32(x):
    """cvt.rna.tf32.f32 on fp32 values: (bits + 0x1000) & 0xFFFFE000 on the magnitude's bits (the sign bit rides
    along, so ties go away from zero for both signs); NaN stays NaN, +-0 stays +-0, and a value within half a TF32
    unit of the largest fp32 rounds to infinity."""
    x = np.asarray(x, np.float32)
    bits = x.view(np.uint32).astype(np.uint64)
    r = ((bits + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)
    return np.where(np.isnan(x), x, r).astype(np.float32)


def _conv64(x, wt, b, s, p):
    """x [B, C, H, W] float64, wt [O, C, k, k] float64 -> [B, O, H', W'] float64 (im2col, one matmul), + b."""
    B, C, H, W = x.shape
    O, _, k, _ = wt.shape
    xp = np.pad(x, ((0, 0), (0, 0), (p, p), (p, p)))
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    cols = np.empty((B, C, k, k, Ho, Wo))
    for kh in range(k):
        for kw in range(k):
            cols[:, :, kh, kw] = xp[:, :, kh: kh + s * (Ho - 1) + 1: s, kw: kw + s * (Wo - 1) + 1: s]
    y = np.einsum("bkhw,ok->bohw", cols.reshape(B, C * k * k, Ho, Wo), wt.reshape(O, -1))
    return y + b[None, :, None, None]


def forward_tf32(row, dims, code, obs):
    """One member's outputs [B, out] (float64) from its formed fp32 parameters ``row``: each layer's weights and
    input rounded with rna_tf32, biases not rounded, products summed in float64, then + bias and the activation
    in float64 (the kernel's arithmetic with exact accumulation)."""
    n_conv = (int(code) >> 24) & 0xff
    shape, convs, linears = unpack(dims, n_conv)
    hidden, tanh_out = HIDDEN[int(code) & 0xff], bool(int(code) & 0x100)
    shapes, _ = layer_shapes(shape, convs, linears)
    row = np.asarray(row, np.float32)
    h, i = np.asarray(obs, np.float32).astype(np.float64), 0
    for li, (ws, bl) in enumerate(shapes):
        wt = rna_tf32(row[i: i + int(np.prod(ws))]).astype(np.float64).reshape(ws)
        i += wt.size
        b = row[i: i + bl].astype(np.float64)
        i += bl
        x = rna_tf32(h.astype(np.float32)).astype(np.float64)
        if li < n_conv:
            h = _act(hidden, _conv64(x, wt, b, convs[li][2], convs[li][3]))
            if li == n_conv - 1:
                h = h.reshape(h.shape[0], -1)
        else:
            h = x @ wt.T + b
            if li + 1 < len(shapes):
                h = _act(hidden, h)
    return np.tanh(h) if tanh_out else h


U32 = 2.0 ** -24
LIPSCHITZ = {"relu": 1.0, "tanh": 1.0, "elu": 1.0, "silu": 1.1, "leaky_relu": 1.0}


def tie_distance(v):
    """Distance of float64 values to the nearest rna_tf32 rounding boundary (halfway between two TF32 values:
    10 explicit significand bits, so the spacing in [2^(e-1), 2^e) is 2^(e-11)); infinite at 0."""
    a = np.abs(np.asarray(v, np.float64))
    _, e = np.frexp(a)
    sp = np.ldexp(1.0, e - 11)
    f = a / sp
    return np.where(a > 0, np.abs(f - np.floor(f) - 0.5) * sp, np.inf)


def forward_tf32_bounds(row, dims, code, obs):
    """forward_tf32, with a bound of the kernel's distance from it per output: (y [B, out] float64, bound [B, out],
    exposed [B, out] bool).  Per layer the kernel's fp32 accumulation adds at most 2 (K + 2) 2^-24 A (A the sum of
    |terms|, K the taps, the bias add included; twice the round-to-nearest bound, since the tensor core's fp32
    accumulation may truncate), the activation 8 half-ulps of |y| (times its Lipschitz constant for what comes in).
    Where a layer input lies within its own error bound of a TF32 rounding boundary, the kernel's fp32 value and
    the model's float64 one may round to neighbouring TF32 values (an operand-rounding flip): that input then adds
    one TF32 spacing times |w| to every output it feeds.  ``exposed`` marks the outputs that such a flip can reach."""
    n_conv = (int(code) >> 24) & 0xff
    shape, convs, linears = unpack(dims, n_conv)
    hidden, tanh_out = HIDDEN[int(code) & 0xff], bool(int(code) & 0x100)
    shapes, _ = layer_shapes(shape, convs, linears)
    row = np.asarray(row, np.float32)
    h, i = np.asarray(obs, np.float32).astype(np.float64), 0
    flip = np.zeros(h.shape)          # the images themselves are exact fp32 operands
    for li, (ws, bl) in enumerate(shapes):
        wt = rna_tf32(row[i: i + int(np.prod(ws))]).astype(np.float64).reshape(ws)
        i += wt.size
        b = row[i: i + bl].astype(np.float64)
        i += bl
        x = rna_tf32(h.astype(np.float32)).astype(np.float64)
        if li < n_conv:
            s, pd = convs[li][2], convs[li][3]
            z = _conv64(x, wt, b, s, pd)
            A = _conv64(np.abs(x), np.abs(wt), np.abs(b), s, pd)
            F = _conv64(flip, np.abs(wt), np.zeros(bl), s, pd)
            K = int(np.prod(ws[1:]))
        else:
            z = x @ wt.T + b
            A = np.abs(x) @ np.abs(wt).T + np.abs(b)
            F = flip @ np.abs(wt).T
            K = ws[1]
        err_z = 2 * (K + 2) * U32 * A + F
        if li == len(shapes) - 1:
            y = np.tanh(z) if tanh_out else z
            return y, err_z + (8 * U32 * np.abs(y) if tanh_out else 0.0), F > 0
        h = _act(hidden, z)
        err_h = LIPSCHITZ[hidden] * err_z + 8 * U32 * np.abs(h)
        _, e = np.frexp(np.abs(h) + err_h)
        flip = np.where(tie_distance(h) <= err_h, np.ldexp(1.0, e - 11), 0.0)
        if li == n_conv - 1:
            h, flip = h.reshape(h.shape[0], -1), flip.reshape(flip.shape[0], -1)


def tau_tf32(y64, target, n_layers):
    """A bound of the kernel's squared-error return against the float64 one: each output within
    e = 2 n_layers 2^-11 max|y| of its row (both operands of each layer rounded, u/2 each), so each term
    (y - t)^2 moves by at most 2|y - t| e + e^2; the mean of that, plus the fp32 sum's own rounding."""
    y = np.asarray(y64, np.float64)
    M = len(y)
    d = (y - np.asarray(target, np.float64)[None]).reshape(M, -1)
    e = 2 * n_layers * 2.0 ** -11 * np.abs(y.reshape(M, -1)).max(1, keepdims=True)
    return (2 * np.abs(d) * e + e * e).mean(1) + (d.shape[1] + 2) * U32 * (d * d).mean(1)


def returns64(y, target, code):
    """Returns of outputs y [M, B, C] in float64: the squared error, the cross-entropy or the accuracy."""
    y, tg = np.asarray(y, np.float64), np.asarray(target, np.float64)
    loss = int(code) & 0xff0000
    if loss == LOSS_ACCURACY:
        return (y.argmax(-1) == tg.argmax(-1)[None]).mean(1)
    if loss == LOSS_XENT:
        m = y.max(-1, keepdims=True)
        lse = m[..., 0] + np.log(np.exp(y - m).sum(-1))
        return -(lse * tg.sum(-1)[None] - (tg[None] * y).sum(-1)).mean(1)
    return -((y - tg[None]) ** 2).mean((1, 2))


class Tf32CnnOracleBackend(CnnOracleBackend):
    """CnnOracleBackend plus ``precision="tf32"`` (forward_tf32, the returns rounded to fp32) and
    ``eval_supports_tf32_cnn``; records the precision of every convolutional evaluate in ``cnn_precisions``."""

    def __init__(self, *a, tf32_supported=True, **k):
        super().__init__(*a, **k)
        self.cnn_precisions = []
        self.tf32_supported = tf32_supported

    def eval_supports_tf32_cnn(self, dims, B, act=0):
        return self.tf32_supported

    def eval_cnn(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                 bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", act=0):
        self.cnn_precisions.append(precision)
        if precision != "tf32":
            return super().eval_cnn(dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus,
                                    ret_minus, bc_plus, bc_minus, bc_obs, bc_dim, precision=precision, act=act)
        assert (act >> 24) & 0xff
        self.cnn_calls += 1
        if offsets is None:
            rows = _np(theta)[None, :]
        else:
            rows, _ = orc.sample_population(_np(theta), _np(table), _np(offsets), sigma)
        y = np.stack([forward_tf32(r, dims, act, _np(obs)) for r in rows])
        rets = returns64(y, _np(target), act).astype(np.float32)
        bcs = y[:, :bc_obs].reshape(len(rows), -1)[:, :bc_dim].astype(np.float32)
        if offsets is None:
            ret_plus[0] = float(rets[0])
            if bc_plus is not None:
                bc_plus.copy_(torch.from_numpy(bcs[0].copy()))
            return
        ret_plus.copy_(torch.from_numpy(rets[:pairs]))
        ret_minus.copy_(torch.from_numpy(rets[pairs:]))
        if bc_plus is not None:
            bc_plus.copy_(torch.from_numpy(bcs[:pairs].copy()))
            bc_minus.copy_(torch.from_numpy(bcs[pairs:].copy()))
