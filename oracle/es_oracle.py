"""CPU restatement (numpy) of the estorch generation hot path.

TEST INFRASTRUCTURE ONLY -- the product (``estorch_b200``) never imports this.

Every function cites the reference lines it restates (paths relative to
``/root/reference``; ``torch/...`` = torch 2.11.0, an *unpinned* third-party
dependency of the reference, ``setup.py:26-31``).

Pinning status
--------------
* ``rank_transformation``: pinned by the reference's only known-answer vector
  (docstring ``estorch/estorch.py:31-35``) -- ``tests/test_oracle.py``.
* everything else (gradient estimate, negate/clamp, Adam, NS/NSR/NSRA blends,
  novelty, NSRA weight schedule, VirtualBatchNorm): the reference ships no test
  vectors, so the restatement is pinned against outputs of the *unmodified*
  reference imported in the build container (``tests/golden/make_golden.py``
  wrote ``tests/golden/*.npz``; the reference is driven through its own
  documented hooks ``_sample_policy`` / ``_calculate_returns``).
* ``noise_offsets`` / ``philox_normal_table`` are definitions of the *new*
  engine (the reference has no noise table, ``estorch.py:187-193`` draws fresh
  RNG); the oracle restates them so the integer path can be compared
  bit-exactly.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import numpy as np

__all__ = [
    "compute_ranks", "center_values", "rank_transformation",
    "mix64", "noise_slots", "noise_offsets", "philox4x32_10", "philox_normal_table",
    "mlp_param_count", "mlp_unflatten", "mlp_forward", "mlp_forward_bf16", "round_bf16", "synthetic_return", "synthetic_bc",
    "round_f16", "mlp_forward_f16",
    "sample_population", "sample_population_bf16s", "evaluate_population",
    "blend_weights", "calculate_grad", "calculate_grad_pairs", "negate_clamp",
    "adam_step", "novelty", "nsra_weight_update", "vbn_stats", "vbn_normalize",
    "conv2d_nchw", "atari_param_layout", "atari_forward",
    "es_generation",
]

# --------------------------------------------------------------------------
# rank transform -- estorch/estorch.py:15-39
# --------------------------------------------------------------------------

def compute_ranks(returns: np.ndarray) -> np.ndarray:
    """``ranks[argsort(r)] = arange(P)`` (estorch.py:22-26), int64.

    The reference uses numpy's default (unstable) argsort, so tie order is
    unspecified there; the engine's rule -- and this oracle's -- is stable by
    member index (``kind='stable'``).  Identical on tie-free input.
    """
    r = np.asarray(returns).reshape(-1)
    ranks = np.empty(r.size, dtype=np.int64)
    ranks[np.argsort(r, kind="stable")] = np.arange(r.size, dtype=np.int64)
    return ranks


def center_values(population_size: int) -> np.ndarray:
    """``arange(P)/(P-1) - 0.5`` in float64 (estorch.py:15-20)."""
    c = np.arange(0, population_size).astype(np.float64)
    c = c / (population_size - 1)
    c -= 0.5
    return c


def rank_transformation(returns) -> np.ndarray:
    """Centred ranks in [-0.5, 0.5], float64 (estorch.py:28-39)."""
    r = np.asarray(returns)
    return center_values(r.size)[compute_ranks(r)]


# --------------------------------------------------------------------------
# noise table addressing (new-engine definition; integer path, bit-exact)
# --------------------------------------------------------------------------
_M64 = (1 << 64) - 1
_GOLD = 0x9E3779B97F4A7C15
_GEN_MUL = 0xD1342543DE82EF95


def mix64(z: int) -> int:
    """splitmix64 finaliser on python ints (mod 2**64)."""
    z = (z + _GOLD) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def noise_slots(table_len: int, n: int) -> int:
    """Number of admissible 32-float-aligned row starts."""
    n_pad = (n + 31) // 32 * 32
    if table_len < n_pad:
        raise ValueError("noise table shorter than one padded parameter row")
    return (table_len - n_pad) // 32 + 1


def noise_offsets(seed: int, gen: int, pair_begin: int, pairs: int,
                  table_len: int, n: int) -> np.ndarray:
    """``off[j] = 32 * (mix64(mix64(seed ^ gen*C) + j) mod nslots)``, int64."""
    nslots = noise_slots(table_len, n)
    base = mix64((seed ^ ((gen * _GEN_MUL) & _M64)) & _M64)
    out = np.empty(pairs, dtype=np.int64)
    for i in range(pairs):
        j = pair_begin + i
        out[i] = 32 * (mix64((base + j) & _M64) % nslots)
    return out


_PHILOX_M0 = 0xD2511F53
_PHILOX_M1 = 0xCD9E8D57
_PHILOX_W0 = 0x9E3779B9
_PHILOX_W1 = 0xBB67AE85


def philox4x32_10(counter_lo: np.ndarray, seed: int) -> Tuple[np.ndarray, ...]:
    """Philox-4x32-10 (Salmon et al. 2011) on counters (c, 0, 0, 0) with key =
    (seed_lo, seed_hi); vectorised over ``counter_lo`` (uint64 array, < 2**64)."""
    c = np.asarray(counter_lo, dtype=np.uint64)
    x0 = (c & np.uint64(0xFFFFFFFF)).astype(np.uint64)
    x1 = (c >> np.uint64(32)).astype(np.uint64)
    x2 = np.zeros_like(x0)
    x3 = np.zeros_like(x0)
    k0 = np.uint64(seed & 0xFFFFFFFF)
    k1 = np.uint64((seed >> 32) & 0xFFFFFFFF)
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(_PHILOX_M0) * x0
        p1 = np.uint64(_PHILOX_M1) * x2
        hi0, lo0 = p0 >> np.uint64(32), p0 & mask
        hi1, lo1 = p1 >> np.uint64(32), p1 & mask
        x0, x1, x2, x3 = (hi1 ^ x1 ^ k0) & mask, lo1, (hi0 ^ x3 ^ k1) & mask, lo0
        k0 = (k0 + np.uint64(_PHILOX_W0)) & mask
        k1 = (k1 + np.uint64(_PHILOX_W1)) & mask
    return x0, x1, x2, x3


def philox_normal_table(length: int, seed: int) -> np.ndarray:
    """Unit normals, fp32: element ``4c+i`` comes from Philox counter ``c``;
    (x0,x1) and (x2,x3) each feed one Box-Muller pair with
    ``u = ((x >> 8) + 0.5) * 2**-24``."""
    if length % 4:
        raise ValueError("table length must be a multiple of 4")
    c = np.arange(length // 4, dtype=np.uint64)
    xs = philox4x32_10(c, seed)
    us = [((x >> np.uint64(8)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)
          for x in xs]
    out = np.empty((length // 4, 4), dtype=np.float32)
    two_pi = np.float32(6.283185307179586)
    for h in range(2):
        r = np.sqrt(np.float32(-2.0) * np.log(us[2 * h])).astype(np.float32)
        ang = (two_pi * us[2 * h + 1]).astype(np.float32)
        out[:, 2 * h] = r * np.cos(ang).astype(np.float32)
        out[:, 2 * h + 1] = r * np.sin(ang).astype(np.float32)
    # estk_fill_noise_table rounds every entry to the nearest fp16-representable value
    # (round-to-nearest-even, like numpy's float32 -> float16), so a 16-bit copy is exact
    return out.reshape(-1).astype(np.float16).astype(np.float32)


# --------------------------------------------------------------------------
# policy forward -- examples/cartpole_es.py:14-20, examples/nsra_es.py:61-67
# --------------------------------------------------------------------------

def mlp_param_count(dims: Sequence[int]) -> int:
    return sum(dims[i + 1] * dims[i] + dims[i + 1] for i in range(len(dims) - 1))


def mlp_unflatten(flat: np.ndarray, dims: Sequence[int]):
    """Split a flat vector in ``parameters_to_vector`` order (weight ``[out,in]``
    row-major, then bias, per Linear; torch/nn/utils/convert_parameters.py:6-25)."""
    layers, idx = [], 0
    for i in range(len(dims) - 1):
        fan_in, fan_out = dims[i], dims[i + 1]
        w = flat[idx: idx + fan_in * fan_out].reshape(fan_out, fan_in)
        idx += fan_in * fan_out
        b = flat[idx: idx + fan_out]
        idx += fan_out
        layers.append((w, b))
    assert idx == flat.shape[0]
    return layers


def mlp_forward(flat: np.ndarray, dims: Sequence[int], obs: np.ndarray) -> np.ndarray:
    """Linear -> ReLU -> ... -> Linear, fp32 (cartpole_es.py:14-20)."""
    h = np.asarray(obs, dtype=np.float32)
    layers = mlp_unflatten(np.asarray(flat, dtype=np.float32), dims)
    for li, (w, b) in enumerate(layers):
        h = (h @ w.T + b).astype(np.float32)
        if li + 1 < len(layers):
            h = np.maximum(h, np.float32(0.0))
    return h


def round_bf16(x: np.ndarray) -> np.ndarray:
    """fp32 -> bf16 (round to nearest even) -> fp32, like cvt.rn.bf16.f32."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    u = (u + np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return u.view(np.float32)


def mlp_forward_bf16(flat: np.ndarray, dims: Sequence[int], obs: np.ndarray) -> np.ndarray:
    """Numerics of the wgmma evaluate path (estk_eval_mlp, ESTK_PREC_BF16): weights and
    layer inputs rounded to bf16, products accumulated in fp32, bias / ReLU in
    fp32.  ``flat`` is the already-perturbed fp32 row."""
    h = round_bf16(np.asarray(obs, dtype=np.float32))
    layers = mlp_unflatten(np.asarray(flat, dtype=np.float32), dims)
    for li, (w, b) in enumerate(layers):
        z = (h.astype(np.float64) @ round_bf16(w).astype(np.float64).T).astype(np.float32) + b
        if li + 1 < len(layers):
            h = round_bf16(np.maximum(z, np.float32(0.0)))
        else:
            h = z.astype(np.float32)
    return h


def round_f16(x: np.ndarray) -> np.ndarray:
    """fp32 -> nearest fp16 (ties to even, saturating at +-65504) -> fp32: the operand
    rounding of the fp16 tensor-core evaluate (cvt.rn.satfinite.f16x2.f32)."""
    return np.clip(np.asarray(x, dtype=np.float32), -65504.0, 65504.0).astype(np.float16).astype(np.float32)


def mlp_forward_f16(flat: np.ndarray, dims: Sequence[int], obs: np.ndarray) -> np.ndarray:
    """Emulation of the roundings of estk_eval_mlp with ESTK_PREC_F16 (test infrastructure for the kernel's
    own arithmetic; parity proper is against mlp_forward): weights and hidden activations
    rounded to fp16, the observation split x_hi + x_lo, fp32 (here fp64) accumulation,
    fp32 bias."""
    x = np.asarray(obs, dtype=np.float32)
    x_hi = round_f16(x)
    h = x_hi.astype(np.float64) + round_f16(x - x_hi).astype(np.float64)
    layers = mlp_unflatten(np.asarray(flat, dtype=np.float32), dims)
    for i, (w, b) in enumerate(layers):
        h = (h @ round_f16(w).astype(np.float64).T + b.astype(np.float64)).astype(np.float32)
        if i + 1 < len(layers):
            h = round_f16(np.maximum(h, 0.0)).astype(np.float64)
    return h.astype(np.float32)


def synthetic_return(out: np.ndarray, target: np.ndarray) -> np.float32:
    """Synthetic agent of SURVEY 8(d): ``-mean((policy(obs) - y)**2)``."""
    d = (out.astype(np.float32) - target.astype(np.float32)).astype(np.float32)
    return np.float32(-np.mean(d * d, dtype=np.float32))


def synthetic_bc(out: np.ndarray, bc_obs: int, bc_dim: int) -> np.ndarray:
    """Behaviour characteristic ``policy(obs[:bc_obs]).flatten()[:bc_dim]``
    (shape of examples/nsra_es.py:45-49: 256 floats)."""
    return np.ascontiguousarray(out[:bc_obs].reshape(-1)[:bc_dim]).astype(np.float32)


# --------------------------------------------------------------------------
# sampling / evaluation -- estorch.py:187-202
# --------------------------------------------------------------------------

def sample_population(theta: np.ndarray, table: np.ndarray, offsets: np.ndarray,
                      sigma: float):
    """(population_parameters, epsilon) as the reference lays them out
    (estorch.py:187-193): rows ``[theta+eps; theta-eps]`` and ``[eps; -eps]``
    with ``eps_j = sigma * T[off_j : off_j+n]`` (the reference's eps carries
    sigma, ``Normal(0, sigma)`` at :189)."""
    n = theta.shape[0]
    t = np.stack([table[o:o + n] for o in offsets]).astype(np.float32)
    eps = (np.float32(sigma) * t).astype(np.float32)
    pop = np.concatenate([theta[None, :] + eps, theta[None, :] - eps]).astype(np.float32)
    return pop, np.concatenate([eps, -eps]).astype(np.float32)


def sample_population_bf16s(theta: np.ndarray, table: np.ndarray, offsets: np.ndarray, sigma: float):
    """Rows as the "bf16s" evaluate path forms them (estk_eval_mlp, ESTK_PREC_BF16S):
    ``W = bf16(theta16 +- sigma16 * eps16)`` with theta16 = bf16(theta), eps16 =
    bf16(T[off:off+n]), sigma16 = bf16(sigma) and ONE rounding of the exact
    product-sum (PTX ``fma.rn.bf16x2``).  Biases are formed from the fp32 sources in
    the kernel -- the caller patches those entries with the exact rows."""
    n = theta.shape[0]
    t16 = np.stack([round_bf16(table[o:o + n]) for o in offsets]).astype(np.float64)
    th16 = round_bf16(theta)[None, :].astype(np.float64)
    s16 = float(round_bf16(np.array([sigma], dtype=np.float32))[0])
    plus = round_bf16((th16 + s16 * t16).astype(np.float32))     # double -> fp32 -> bf16 (double rounding is rare)
    minus = round_bf16((th16 - s16 * t16).astype(np.float32))
    return np.concatenate([plus, minus]).astype(np.float32)


def evaluate_population(pop: np.ndarray, dims, obs, target,
                        bc_obs: int = 0, bc_dim: int = 0):
    """Per-row rollout of the synthetic agent (estorch.py:195-202)."""
    rets = np.empty(pop.shape[0], dtype=np.float32)
    bcs = np.empty((pop.shape[0], bc_dim), dtype=np.float32) if bc_dim else None
    for i in range(pop.shape[0]):
        out = mlp_forward(pop[i], dims, obs)
        rets[i] = synthetic_return(out, target)
        if bc_dim:
            bcs[i] = synthetic_bc(out, bc_obs, bc_dim)
    return rets, bcs


# --------------------------------------------------------------------------
# gradient estimate -- estorch.py:174-179, :419-425, :542-549, :640-648
# --------------------------------------------------------------------------

def blend_weights(returns: np.ndarray, algo: str = "es", weight: float = 1.0) -> np.ndarray:
    """fp32 row vector multiplied into epsilon.

    es   : c(reward)                              (estorch.py:175-176)
    ns   : c(novelty)                             (:420-422)
    nsr  : (c(novelty) + c(reward)) / 2           (:543-547)
    nsra : w*c(reward) + (1-w)*c(novelty)         (:641-646)
    ``returns`` is ``[P]`` (es) or ``[P,2]`` = (reward, novelty) (:441).
    """
    r = np.asarray(returns, dtype=np.float32)
    if algo == "es":
        return rank_transformation(r.reshape(-1)).astype(np.float32)
    c_rew = rank_transformation(r[:, 0]).astype(np.float32)
    c_nov = rank_transformation(r[:, 1]).astype(np.float32)
    if algo == "ns":
        return c_nov
    if algo == "nsr":
        return ((c_nov + c_rew) / np.float32(2.0)).astype(np.float32)
    if algo == "nsra":
        w = np.float32(weight)
        one_minus = np.float32(1.0 - weight)
        return (w * c_rew + one_minus * c_nov).astype(np.float32)
    raise ValueError(algo)


def calculate_grad(returns, epsilon: np.ndarray, sigma: float, algo="es", weight=1.0):
    """Reference form: ``(c[1xP] @ E[Pxn]) / (P*sigma)`` (estorch.py:177-178)."""
    c = blend_weights(returns, algo, weight)
    P = epsilon.shape[0]
    g = (c[None, :].astype(np.float32) @ epsilon.astype(np.float32)).reshape(-1)
    return (g / np.float32(P * sigma)).astype(np.float32)


def calculate_grad_pairs(returns, table, offsets, n, algo="es", weight=1.0):
    """Pair-difference form on the unit-normal rows, in float64 (the
    well-conditioned evaluation of the same sum; SURVEY App. A.1):
    ``g = (1/P) * sum_j (c_j - c_{j+pairs}) * T[off_j : off_j+n]``."""
    c = blend_weights(returns, algo, weight).astype(np.float64)
    pairs = len(offsets)
    acc = np.zeros(n, dtype=np.float64)
    for j, o in enumerate(offsets):
        acc += (c[j] - c[j + pairs]) * table[o:o + n].astype(np.float64)
    return acc / (2 * pairs)


def negate_clamp(grad: np.ndarray) -> np.ndarray:
    """``param.grad = -grad[slice]; clamp_(-1, 1)`` (estorch.py:236-244)."""
    return np.clip(-grad.astype(np.float32), np.float32(-1.0), np.float32(1.0))


# --------------------------------------------------------------------------
# optimizer -- estorch.py:245 -> torch/optim/adam.py:457,476,529-546
# --------------------------------------------------------------------------

def adam_step(theta, m, v, grad, step: int, lr=0.01, beta1=0.9, beta2=0.999,
              eps=1e-8, weight_decay=0.0):
    """torch.optim.Adam single-tensor CPU path, defaults as in
    examples/cartpole_es.py:48-50.  ``step`` is the 1-based step count *after*
    the increment.  Returns new (theta, m, v), fp32."""
    f = np.float32
    g = grad.astype(np.float32)
    if weight_decay:
        g = (g + f(weight_decay) * theta).astype(np.float32)
    m = (m + (g - m) * f(1.0 - beta1)).astype(np.float32)          # lerp_
    v = (v * f(beta2)).astype(np.float32)
    v = (v + (f(1.0 - beta2) * g) * g).astype(np.float32)          # addcmul_
    bc1 = 1.0 - beta1 ** step
    bc2 = 1.0 - beta2 ** step
    step_size = lr / bc1
    denom = (np.sqrt(v).astype(np.float32) / f(math.sqrt(bc2)) + f(eps)).astype(np.float32)
    theta = (theta + (f(-step_size) * m) / denom).astype(np.float32)  # addcdiv_
    return theta, m, v


# --------------------------------------------------------------------------
# novelty search pieces -- estorch.py:412-417, :650-662
# --------------------------------------------------------------------------

def novelty(bc: np.ndarray, archive: np.ndarray, k: int) -> float:
    """``sum(k nearest euclidean distances) / ||archive||_F`` (estorch.py:412-417;
    cKDTree.query pads with inf when the archive has < k points and the
    reference drops those, :415).  Brute force, float64 like scipy."""
    a = np.asarray(archive, dtype=np.float64)
    d = np.sqrt(((a - np.asarray(bc, dtype=np.float64)[None, :]) ** 2).sum(axis=1))
    d.sort()
    return float(d[:k].sum() / np.linalg.norm(a))


def nsra_weight_update(weight, t, episode_reward, best_reward,
                       weight_t, min_weight=0.0, weight_delta=0.05):
    """NSRA ``_after_optimize`` schedule (estorch.py:650-662).  The reference
    hard-codes ``weight_delta = 0.05`` (:637).  Returns (weight, t, best_reward)."""
    if episode_reward > best_reward:
        return min(weight + weight_delta, 1.0), 0, episode_reward
    t += 1
    if t >= weight_t:
        return max(weight - weight_delta, min_weight), 0, best_reward
    return weight, t, best_reward


# --------------------------------------------------------------------------
# VirtualBatchNorm + Atari conv policy -- estorch/modules.py:42-58,
# examples/atari.py:14-37
# --------------------------------------------------------------------------

def vbn_stats(xref: np.ndarray):
    """Per-(C,H,W) mean and *unbiased* variance over the batch dim
    (modules.py:51-52: ``torch.mean(x,0,keepdim)``, ``torch.var(x,0,keepdim)``)."""
    x = xref.astype(np.float32)
    mean = x.mean(axis=0, keepdims=True, dtype=np.float32)
    var = x.var(axis=0, keepdims=True, ddof=1, dtype=np.float32)
    return mean.astype(np.float32), var.astype(np.float32)


def vbn_normalize(x, mean, var, gamma, beta, eps=1e-5):
    """``(x-mean)/sqrt(var+eps) * gamma[c] + beta[c]`` (modules.py:42-46)."""
    C = gamma.shape[0]
    y = (x - mean) / np.sqrt(var + np.float32(eps))
    return (y * gamma.reshape(1, C, 1, 1) + beta.reshape(1, C, 1, 1)).astype(np.float32)


def conv2d_nchw(x, w, b, stride):
    """Valid cross-correlation, NCHW / OIHW (torch.nn.Conv2d semantics)."""
    N, C, H, W = x.shape
    O, _, KH, KW = w.shape
    OH, OW = (H - KH) // stride + 1, (W - KW) // stride + 1
    cols = np.empty((N, OH, OW, C * KH * KW), dtype=np.float32)
    for i in range(OH):
        for j in range(OW):
            patch = x[:, :, i * stride:i * stride + KH, j * stride:j * stride + KW]
            cols[:, i, j, :] = patch.reshape(N, -1)
    y = cols.reshape(-1, C * KH * KW) @ w.reshape(O, -1).T + b
    return y.reshape(N, OH, OW, O).transpose(0, 3, 1, 2).astype(np.float32)


def atari_param_layout(n_actions: int):
    """Registration order of examples/atari.py:17-23 (SURVEY App. A.10)."""
    return [("conv1.w", (16, 4, 8, 8)), ("conv1.b", (16,)), ("bn1.w", (16,)), ("bn1.b", (16,)),
            ("conv2.w", (32, 16, 4, 4)), ("conv2.b", (32,)), ("bn2.w", (32,)), ("bn2.b", (32,)),
            ("fc1.w", (256, 2592)), ("fc1.b", (256,)), ("fc2.w", (n_actions, 256)),
            ("fc2.b", (n_actions,))]


def atari_forward(flat, n_actions, xref, x):
    """Policy.forward of examples/atari.py:25-37: the reference batch runs
    through conv1/bn1/conv2/bn2 first (stats), then the real batch."""
    p, idx = {}, 0
    for name, shape in atari_param_layout(n_actions):
        sz = int(np.prod(shape))
        p[name] = flat[idx:idx + sz].reshape(shape).astype(np.float32)
        idx += sz
    r1 = conv2d_nchw(xref, p["conv1.w"], p["conv1.b"], 4)
    m1, v1 = vbn_stats(r1)
    r1 = np.maximum(vbn_normalize(r1, m1, v1, p["bn1.w"], p["bn1.b"]), 0)
    r2 = conv2d_nchw(r1, p["conv2.w"], p["conv2.b"], 2)
    m2, v2 = vbn_stats(r2)
    h = conv2d_nchw(x, p["conv1.w"], p["conv1.b"], 4)
    h = np.maximum(vbn_normalize(h, m1, v1, p["bn1.w"], p["bn1.b"]), 0)
    h = conv2d_nchw(h, p["conv2.w"], p["conv2.b"], 2)
    h = np.maximum(vbn_normalize(h, m2, v2, p["bn2.w"], p["bn2.b"]), 0)
    h = h.reshape(-1, 2592)
    h = np.maximum(h @ p["fc1.w"].T + p["fc1.b"], 0).astype(np.float32)
    return (h @ p["fc2.w"].T + p["fc2.b"]).astype(np.float32)


# --------------------------------------------------------------------------
# one whole generation -- estorch.py:214-248
# --------------------------------------------------------------------------

def es_generation(theta, m, v, step, table, offsets, sigma, dims, obs, target,
                  lr=0.01, beta1=0.9, beta2=0.999, eps=1e-8, returns=None):
    """sample -> evaluate -> rank -> mm -> negate/clamp -> Adam -> post-update
    rollout, for the classic ES on the synthetic agent.  ``returns`` may be
    injected (stage-B parity: gradient on identical return bits)."""
    pop, epsilon = sample_population(theta, table, offsets, sigma)
    if returns is None:
        returns, _ = evaluate_population(pop, dims, obs, target)
    ranks = compute_ranks(returns)
    grad = calculate_grad(returns, epsilon, sigma)
    g = negate_clamp(grad)
    theta1, m1, v1 = adam_step(theta, m, v, g, step + 1, lr, beta1, beta2, eps)
    episode_reward = synthetic_return(mlp_forward(theta1, dims, obs), target)
    return dict(returns=returns, ranks=ranks, grad=grad, theta=theta1, m=m1, v=v1,
                episode_reward=episode_reward)
