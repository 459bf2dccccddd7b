"""TEST-ONLY: the 16-bit tensor-core MLP evaluate (estk_eval_mlp_tc.cu, estk_eval_mlp_tc_stream.cu) restated in
float64, with a bound of each kernel output's distance from the restatement.

The modes, as the kernels compute them:
    f16 (and f16_any)  W16 = rn_f16(fmaf(s*sigma, eps, theta)): one fp32 fma, then fp16 with satfinite; layer 0
                       takes x_hi = rn_f16(x) and x_lo = rn_f16(x - x_hi) (fp32 subtraction) on the same weights,
                       x_hi saturating, x_lo not: an infinity, or a finite |x| >= 131024, enters with x_lo = +-inf
                       (its outputs are non-finite, as an infinity's are in fp32)
    bf16               W16 = rn_bf16(fmaf(s*sigma, eps, theta)); layer 0 takes rn_bf16(x)
    bf16s              W16 = rn_bf16(theta16 + sigma16 * eps16), the exact value rounded once (fma.rn.bf16x2), from
                       the bf16 shadows of theta, the table row and +-sigma; layer 0 as bf16
Every mode forms the biases as fmaf(s*sigma, eps, theta) in fp32 and accumulates in fp32.  A hidden layer's fp32
activation (``orc.HIDDEN``'s kinds) is rounded once to the 16-bit type (fp16 with satfinite); the last layer is
fp32, then the optional fp32 tanh.

``forward`` works on formed rows (``form``) and keeps the accumulation exact.  Its bound follows
``_cnn_tf32_oracle.forward_tf32_bounds``: per layer 2 (K + 2) 2^-24 A for the fp32 accumulation (A the sum of
|terms|, K the row's non-zero inputs times the operands per input, bias add included; twice round-to-nearest,
since the tensor core may truncate), the
activation's own ulps, and for every 16-bit input whose value the kernel may round to another 16-bit neighbour
(its error interval straddles a rounding boundary: an operand flip) the size of that flip times |w|; the outputs a
flip can reach are ``exposed``.  fp16 operands below 2^-14 add 2^-24 |other operand|.

Everything is torch.float64 on the device of the arguments (cuBLAS on a GPU, not code under test)."""
import numpy as np
import torch

import _mlp_oracle as mlp
from oracle import es_oracle as orc

U32 = 2.0 ** -24
F16_MAX = 65504.0
F16_MIN_NORMAL = 2.0 ** -14
SIG_BITS = {"f16": 11, "bf16": 8}
# half-ulps (2^-24 |a|) of the device's fp32 activation against the float64 one (tanhf, expf, expm1f are within 2
# ulps, SiLU adds its sum and divide); LeakyReLU rounds y * 0.01f once
ACT_HALF_ULPS = {"relu": 0.0, "leaky_relu": 1.0, "tanh": 16.0, "elu": 16.0, "silu": 16.0}
LIPSCHITZ = {"relu": 1.0, "tanh": 1.0, "elu": 1.0, "silu": 1.1, "leaky_relu": 1.0}
LEAKY = float(np.float32(0.01))


def kind(mode):
    """The 16-bit operand type of a mode."""
    return "f16" if mode in ("f16", "f16_any") else "bf16"


def t64(x, device="cpu"):
    return torch.as_tensor(np.asarray(x), device=device).to(torch.float64)


def spacing(x, typ):
    """The ``typ`` spacing at float64 values x: 2^(e - s) for |x| in [2^(e-1), 2^e), s the significand bits; fp16
    subnormals 2^-24."""
    _, e = torch.frexp(x)
    return pow2((e - SIG_BITS[typ]).clamp(min=-24 if typ == "f16" else -133))


def pow2(e):
    """2^e as float64, exactly, for integer tensors e in [-1022, 1023]: the exponent field itself (torch.pow on a
    CUDA device is the libm pow, which need not return powers of two exactly)."""
    return ((e.to(torch.int64) + 1023) << 52).view(torch.float64)


def rn16(x, typ):
    """float64 -> the nearest ``typ`` ("f16" or "bf16") value, ties to even, as float64; f16 saturates at +-65504
    (satfinite: +-inf too) and has subnormals down to 2^-24.  One rounding from the float64 value."""
    q = spacing(x, typ)
    r = torch.where(torch.isfinite(x), torch.round(x / q) * q, x)
    return r.clamp(-F16_MAX, F16_MAX) if typ == "f16" else r


def fl32(x):
    return x.to(torch.float32).to(torch.float64)


def fma32(a, b, c):
    """fp32 fma(a, b, c) of fp32 values held in float64, rounded once: the product is exact in float64 and the
    float64 sum is rounded to odd (``orc.fma32``), which then rounds to the correctly rounded fp32 result."""
    p = a * b
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)
    inexact = (err != 0) & torch.isfinite(err) & ((s.view(torch.int64) & 1) == 0)
    s = torch.where(inexact, torch.nextafter(s, torch.where(err > 0, torch.inf, -torch.inf).to(s)), s)
    return fl32(s)


def layout(dims):
    """[(K, N, weight slice, bias slice)] of a flat parameter row."""
    out, i = [], 0
    for K, N in zip(dims[:-1], dims[1:]):
        out.append((K, N, slice(i, i + K * N), slice(i + K * N, i + K * N + N)))
        i += K * N + N
    return out


def is_weight(dims, device="cpu"):
    w = torch.zeros(orc.mlp_param_count(dims), dtype=torch.bool, device=device)
    for _, _, ws, _ in layout(dims):
        w[ws] = True
    return w


def form(mode, dims, theta, table, offsets, sigma, centre=False, device="cpu", exact=False):
    """The members' formed rows [M, n] float64: the 16-bit weights and the fp32 biases, members ordered
    [+ for each offset, - for each offset] (then theta itself with ``centre``); ``exact``: the fp32 rows
    fmaf(s*sigma, eps, theta) themselves, weights not rounded."""
    theta = t64(np.asarray(theta, np.float32), device)
    eps = t64(np.stack([table[o:o + theta.numel()] for o in offsets]).astype(np.float32), device)
    ssig = t64(np.array([sigma, -sigma], np.float32), device)
    s = ssig.repeat_interleave(len(offsets))[:, None]
    e = eps.repeat(2, 1)
    if centre:
        s = torch.cat([s, torch.zeros(1, 1, dtype=s.dtype, device=device)])
        e = torch.cat([e, torch.zeros_like(e[:1])])
    f = fma32(s, e, theta[None])
    if exact:
        return f
    typ = kind(mode)
    if mode == "bf16s":
        w16 = rn16(rn16(theta, typ)[None] + rn16(s, typ) * rn16(e, typ), typ)
    else:
        w16 = rn16(f, typ)
    return torch.where(is_weight(dims, device)[None], w16, f)


def layer0(mode, obs):
    """Layer 0's 16-bit operands [B, K0], each multiplied by the same weights: [x_hi, x_lo] in fp16, [rn_bf16(x)]."""
    typ = kind(mode)
    x = obs if torch.is_tensor(obs) else t64(np.asarray(obs, np.float32))
    hi = rn16(x, typ)
    if typ == "bf16":
        return [hi]
    d = fl32(x - hi)                    # x_lo is rounded without satfinite: beyond 65520 it is +-inf
    return [hi, torch.where(d.abs() >= 65520.0, d * torch.inf, rn16(d, typ))]


def act64(hidden, z):
    """The hidden activation in float64."""
    if hidden == "relu":
        return z.clamp(min=0.0)
    if hidden == "tanh":
        return torch.tanh(z)
    if hidden == "elu":
        return torch.where(z > 0, z, torch.expm1(z))
    if hidden == "silu":
        return z / (1.0 + torch.exp(-z))
    return torch.where(z > 0, z, z * LEAKY)


def _sub(v):
    return ((v != 0) & (v.abs() < F16_MIN_NORMAL)).to(v.dtype)


def forward(mode, rows, dims, ops, code):
    """Outputs of formed rows [M, n] on layer-0 operands ``ops`` (``layer0``): (y [M, B, out], bound, exposed), the
    kernel's outputs within ``bound`` of y.  Non-finite inputs give non-finite bounds."""
    hidden, output, _ = mlp.decode(code)
    typ = kind(mode)
    M = rows.shape[0]
    flip = None
    for li, (K, N, ws, bs) in enumerate(layout(dims)):
        W = rows[:, ws].reshape(M, N, K).transpose(1, 2)          # [M, K, N]
        Wa = W.abs()
        b = rows[:, bs][:, None, :]
        z = sum(o @ W for o in ops) + b
        A = sum(o.abs() @ Wa for o in ops) + b.abs()
        # the products that are not exactly zero: an fp32 accumulator adding an exact zero does not round
        nz = sum((o != 0).to(o.dtype).sum(-1, keepdim=True) for o in ops)
        err = 2 * (nz + 2) * U32 * A
        if flip is not None:
            err = err + flip @ Wa
        if typ == "f16":
            err = err + U32 * sum(_sub(o) @ Wa + o.abs() @ _sub(W) for o in ops)
        if li == len(dims) - 2:
            y = torch.tanh(z) if output == "tanh" else z
            bound = err + 16 * U32 * y.abs() if output == "tanh" else err
            exposed = (flip @ Wa > 0) if flip is not None else torch.zeros_like(y, dtype=torch.bool)
            return y, bound, exposed
        a = act64(hidden, z)
        ea = LIPSCHITZ[hidden] * err + ACT_HALF_ULPS[hidden] * U32 * a.abs()
        h = rn16(a, typ)
        flip = torch.maximum(rn16(a + ea, typ) - h, h - rn16(a - ea, typ))
        ops = [h]


def bound_exact(mode, rows32, dims, obs, code):
    """The float64 forward of exact fp32 rows [M, n] (no 16-bit rounding) and a first-order bound of the 16-bit
    kernel's distance from it: every operand rounded (2^-s relative, s the type's significand bits with the hidden
    one; fp16 also 2^-24 absolute for subnormals; the fp16 observations carry ~22 bits as x_hi + x_lo) and the fp32
    accumulation, carried through |W| and the activation's Lipschitz constant.  A looser bar than ``forward``'s."""
    hidden, output, _ = mlp.decode(code)
    f16 = kind(mode) == "f16"
    u, sub = 2.0 ** -SIG_BITS[kind(mode)], (U32 if f16 else 0.0)
    M = rows32.shape[0]
    h = obs if torch.is_tensor(obs) else t64(np.asarray(obs, np.float32), rows32.device)
    e_in = (2.0 ** -21 * h.abs() + sub) if f16 else u * h.abs()
    for li, (K, N, ws, bs) in enumerate(layout(dims)):
        W = rows32[:, ws].reshape(M, N, K).transpose(1, 2)
        b = rows32[:, bs][:, None, :]
        Wa = W.abs()
        ew = u * Wa + sub
        z = h @ W + b
        err = e_in @ (Wa + ew) + h.abs() @ ew + 2 * (2 * K + 2) * U32 * ((h.abs() + e_in) @ (Wa + ew) + b.abs())
        if li == len(dims) - 2:
            y = torch.tanh(z) if output == "tanh" else z
            return y, err + (16 * U32 * y.abs() if output == "tanh" else 0.0)
        h = act64(hidden, z)
        e_in = LIPSCHITZ[hidden] * err + (u + ACT_HALF_ULPS[hidden] * U32) * h.abs() + sub
        if f16:                                            # saturated at 65504: no first-order bound
            e_in = torch.where(h.abs() > F16_MAX, torch.inf, e_in)


def returns64(Y, target, code):
    """Returns of given fp32 outputs Y [M, B, C] in float64, and a bound of the kernel's fp32 reduction of them:
    (r [M], bound [M]).  Squared error: each term (y - t)^2 from one fp32 subtraction and one fma, summed in any
    order, then one divide: (n + 4) 2^-24 mean((y - t)^2) over n = B C terms.  Cross-entropy: per row the max, the
    sum of expf (2 ulps each) and logf, the fma chains of sum t*y and sum t, then the sum over rows and the divide;
    each step's worst case, doubled.  Accuracy: exact (count / B, the first index of each row's maximum)."""
    Y = Y.to(torch.float64)
    t = target.to(torch.float64)
    M, B, C = Y.shape
    loss = int(code) & 0xff0000
    if loss == mlp.LOSS_ACCURACY:
        # one IEEE fp32 divide, in numpy: torch divides by a scalar as a product with its reciprocal
        hit = (Y.argmax(-1) == t.argmax(-1)[None]).sum(1).cpu().numpy().astype(np.float32)
        return t64(hit / np.float32(B), Y.device), torch.zeros(M, dtype=torch.float64, device=Y.device)
    if loss == mlp.LOSS_XENT:
        m = Y.amax(-1, keepdim=True)
        lse = m[..., 0] + torch.log(torch.exp(Y - m).sum(-1))
        st, sty = t.sum(-1)[None], (t[None] * Y).sum(-1)
        sta = (t[None] * Y).abs().sum(-1)
        ce = lse * st - sty
        eb = ((C + 10) + (C + 5) * lse.abs()) * U32 * st + (C + 2) * U32 * sta
        bound = 2 * ((eb.sum(1) + (B + 2) * U32 * ce.abs().sum(1)) / B + U32 * (ce.sum(1) / B).abs())
        return -ce.mean(1), bound
    d2 = ((Y - t[None]) ** 2).reshape(M, -1)
    return -d2.mean(1), (d2.shape[1] + 4) * U32 * d2.mean(1)
