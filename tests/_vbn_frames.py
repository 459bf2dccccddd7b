"""TEST-ONLY: Atari-like frames for the VirtualBatchNorm tests, and a float64 forward of the conv + VBN policy of
the reference's Atari example (examples/atari.py:14-37) to hold the kernels against.

The reference builds its frames from the Y channel of the screen without dividing by 255, so pixels run from 0 to
255, and most of the screen (walls, score bar, background) is the same in every frame of the reference batch.
VBN's statistics are hard there: the mean is large and the variance small or exactly zero.  Every generator here is
deterministic from its seed and returns ``(xref [R,4,84,84], obs [B,4,84,84])`` float32:

  raw      constant grey background (142), a static wall and score bar, two small moving bright objects that
           stay in the lower-left part of the screen, so the rest is constant over the reference batch;
  unit     the same frames divided by 255;
  near     raw, plus +-1..2 grey levels of noise on a constant region (a near-zero, non-zero variance);
  same     all R reference frames identical: the true variance is exactly 0 everywhere;
  outlier  reference frame 0 carries objects where every other reference frame is constant.

Observations always differ from the reference batch at positions that are constant in it (a ball in the
upper half, a brick knocked out of the wall), which is where a wrong VBN scale is multiplied by a large
difference."""
import numpy as np
import torch
from numpy.lib.stride_tricks import sliding_window_view

from oracle import es_oracle as orc
from _pop_conv_oracle import AtariPolicy

f32, f64 = np.float32, np.float64
KINDS = ("raw", "unit", "near", "same", "outlier")
BG, WALL, BRIGHT = 142.0, 200.0, 255.0
EPS = 1e-5
P1, P2 = 16 * 20 * 20, 32 * 9 * 9


def _screen():
    """The static part of every frame: background, score bar (rows 0-5), a brick wall (rows 16-27)."""
    s = np.full((84, 84), BG, dtype=f64)
    s[0:6, :] = 0.0
    s[16:28, 4:80] = WALL
    s[16:28, 4:80:8] = 170.0              # gaps between bricks
    return s


def _stack(screen, objects):
    """Four stacked frames; each object (row, col, h, w, dr, dc, value) moves by (dr, dc) per frame."""
    x = np.repeat(screen[None], 4, axis=0)
    for r, c, h, w, dr, dc, v in objects:
        for t in range(4):
            rr, cc = int(np.clip(r + t * dr, 0, 84 - h)), int(np.clip(c + t * dc, 0, 84 - w))
            x[t, rr:rr + h, cc:cc + w] = v
    return x


def _moving(rng, n, rows, cols):
    """n small bright objects inside rows x cols, with per-frame motion of up to 2 pixels."""
    out = []
    for _ in range(n):
        h, w = int(rng.randint(2, 4)), int(rng.randint(2, 5))
        out.append((int(rng.randint(*rows)), int(rng.randint(*cols)), h, w, int(rng.randint(-2, 3)),
                    int(rng.randint(-2, 3)), BRIGHT if rng.rand() < 0.5 else 90.0))
    return out


def _obs(rng, B, screen):
    """Observations: objects anywhere, including the regions constant over the reference batch, and a brick
    knocked out of the wall."""
    frames = []
    for _ in range(B):
        s = screen.copy()
        c = int(rng.randint(0, 10)) * 8 + 4
        s[16 + 4 * int(rng.randint(0, 3)):20 + 4 * int(rng.randint(0, 3)) + 4, c:c + 8] = BG
        frames.append(_stack(s, _moving(rng, 2, (6, 82), (0, 82)) + [(int(rng.randint(30, 60)), int(rng.randint(40, 80)),
                                                                      2, 2, 1, -1, BRIGHT)]))
    return np.stack(frames)


def frames(kind, R, B, seed=0):
    """(xref [R,4,84,84], obs [B,4,84,84]) float32 of one of KINDS."""
    assert kind in KINDS, kind
    rng = np.random.RandomState(seed)
    screen = _screen()
    if kind == "same":
        one = _stack(screen, _moving(rng, 2, (40, 80), (0, 44)))
        xref = np.repeat(one[None], R, axis=0)
    elif kind == "outlier":
        xref = np.repeat(screen[None, None], R, axis=0).repeat(4, axis=1)
        xref[0] = _stack(screen, _moving(rng, 4, (6, 82), (0, 82)))
    else:
        xref = np.stack([_stack(screen, _moving(rng, 2, (40, 80), (0, 44))) for _ in range(R)])
        if kind == "near":
            xref[:, :, 30:84, 44:84] += rng.randint(-2, 3, size=(R, 4, 54, 40))
    obs = _obs(rng, B, screen)
    if kind == "unit":
        return (xref.astype(f32) / f32(255)).astype(f32), (obs.astype(f32) / f32(255)).astype(f32)
    return xref.astype(f32), obs.astype(f32)


def policy_row(n_actions, theta, seed):
    """Flat parameters of the policy: torch's initialisation ("init"), or with VBN gamma / beta moved by
    0.2 N(0, 1) as training moves them ("trained")."""
    torch.manual_seed(seed)
    pol = AtariPolicy(n_actions, None)
    if theta == "trained":
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for name, p_ in pol.named_parameters():
                if name.startswith("bn"):
                    p_.add_(0.2 * torch.randn(p_.shape, generator=g))
    return torch.nn.utils.parameters_to_vector(pol.parameters()).detach().numpy()


# ---------------------------------------------------------------- float64 forward
def unflatten64(row, n_actions):
    p, idx = {}, 0
    for name, shape in orc.atari_param_layout(n_actions):
        sz = int(np.prod(shape))
        p[name] = np.asarray(row[idx:idx + sz], dtype=f64).reshape(shape)
        idx += sz
    return p


def conv64(x, w, b, stride):
    """Valid cross-correlation in float64, x [N,C,H,W], w [O,C,k,k] -> [N,O,OH,OW]."""
    k = w.shape[-1]
    v = sliding_window_view(np.asarray(x, dtype=f64), (k, k), axis=(2, 3))[:, :, ::stride, ::stride]
    return np.einsum("nchwij,ocij->nohw", v, w, optimize=True) + b[None, :, None, None]


def _moments(y):
    """Two-pass mean and unbiased variance over the batch axis (torch.var_mean, estorch/modules.py:51-52)."""
    mean = y.mean(axis=0, keepdims=True)
    var = ((y - mean) ** 2).sum(axis=0, keepdims=True) / (y.shape[0] - 1)
    return mean, var


def _vbn(x, mean, var, g, b):
    """(x - mean) / sqrt(var + eps) * gamma + beta (estorch/modules.py:42-46)."""
    return (x - mean) / np.sqrt(var + EPS) * g[None, :, None, None] + b[None, :, None, None]


class Forward64:
    """The policy of one member row (fp32 values, promoted) in float64.  ``stats`` holds the VBN statistics of
    both layers, (mean, var) per (C, H, W) position, and ``folded()`` what the kernels store, the scale
    a = gamma / sqrt(var + eps) and the mean, in their layout [a1, mean1, a2, mean2]."""

    def __init__(self, row, n_actions, xref):
        self.p = p = unflatten64(row, n_actions)
        r1 = conv64(xref, p["conv1.w"], p["conv1.b"], 4)
        m1, v1 = _moments(r1)
        h = np.maximum(_vbn(r1, m1, v1, p["bn1.w"], p["bn1.b"]), 0)
        r2 = conv64(h, p["conv2.w"], p["conv2.b"], 2)
        m2, v2 = _moments(r2)
        self.stats = ((m1, v1), (m2, v2))

    def __call__(self, x):
        p, ((m1, v1), (m2, v2)) = self.p, self.stats
        h = np.maximum(_vbn(conv64(x, p["conv1.w"], p["conv1.b"], 4), m1, v1, p["bn1.w"], p["bn1.b"]), 0)
        h = np.maximum(_vbn(conv64(h, p["conv2.w"], p["conv2.b"], 2), m2, v2, p["bn2.w"], p["bn2.b"]), 0)
        h = np.maximum(h.reshape(h.shape[0], 2592) @ p["fc1.w"].T + p["fc1.b"], 0)
        return h @ p["fc2.w"].T + p["fc2.b"]

    def folded(self):
        out = []
        for (mean, var), g in zip(self.stats, ("bn1.w", "bn2.w")):
            a = self.p[g][None, :, None, None] / np.sqrt(var + EPS)
            out += [a.reshape(-1), mean.reshape(-1)]
        return np.concatenate(out)


def reference32(row, n_actions, xref, x):
    """The reference's fp32 arithmetic: the policy in torch float32 on the CPU with this package's
    VirtualBatchNorm (torch.var_mean statistics).  Returns (outputs [B, A], folded statistics in the kernels'
    layout); their distance from float64 is the floor any fp32 implementation is measured against."""
    pol = AtariPolicy(n_actions, torch.from_numpy(np.ascontiguousarray(xref, dtype=f32)))
    torch.nn.utils.vector_to_parameters(torch.from_numpy(np.asarray(row, dtype=f32).copy()), pol.parameters())
    F = torch.nn.functional
    with torch.no_grad():
        F.relu(pol.bn2(pol.conv2(F.relu(pol.bn1(pol.conv1(pol.xref))))))
        folded = []
        for bn in (pol.bn1, pol.bn2):
            var, mean = bn._ref_stats
            a = bn.weight.view(1, -1, 1, 1) / torch.sqrt(var + bn.eps)
            folded += [a.reshape(-1), mean.reshape(-1)]
            bn._ref_stats = None
        out = pol(torch.from_numpy(np.ascontiguousarray(x, dtype=f32)))
    return out.numpy().astype(f64), torch.cat(folded).numpy().astype(f64)


def stats_slices():
    """(name, slice) of the four parts of a member's folded statistics."""
    return (("a1", slice(0, P1)), ("mean1", slice(P1, 2 * P1)), ("a2", slice(2 * P1, 2 * P1 + P2)),
            ("mean2", slice(2 * P1 + P2, 2 * P1 + 2 * P2)))


def scale_err(got, want):
    """Largest elementwise relative error of a VBN scale (a > 0 everywhere)."""
    return float(np.max(np.abs(np.asarray(got, f64) - want) / np.abs(want)))


def rel_err(a, b):
    """max|a - b| / max|b|, the project's tolerance measure."""
    a, b = np.asarray(a, dtype=f64), np.asarray(b, dtype=f64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


# ---------------------------------------------------------------- the one-pass statistics, emulated
def conv1_fp32_chain(x, w, b):
    """conv1 as the fp32 kernels compute it: one fmaf chain per output from the bias in (ci, kh, kw) order.
    x [N,4,84,84], w [16,4,8,8], b [16] float32 -> [N,16,20,20] float32."""
    v = sliding_window_view(np.asarray(x, dtype=f32), (8, 8), axis=(2, 3))[:, :, ::4, ::4]   # [N,4,20,20,8,8]
    v = v.transpose(0, 2, 3, 1, 4, 5).reshape(x.shape[0], 1, 20, 20, 256)
    w = np.asarray(w, dtype=f32).reshape(1, 16, 1, 1, 256)
    acc = np.broadcast_to(np.asarray(b, dtype=f32).reshape(1, 16, 1, 1), (x.shape[0], 16, 20, 20)).copy()
    for k in range(256):
        acc = orc.fma32(v[..., k], w[..., k], acc)
    return acc


def vbn1_scale_one_pass(y, gamma):
    """The fp32 kernels' layer-1 scale before accurate statistics: sum and fmaf sum of squares in frame order,
    var = max((ssq - sum * mean) / (R - 1), 0), a = gamma / sqrtf(var + 1e-5f)."""
    R = y.shape[0]
    s = np.zeros(y.shape[1:], f32)
    q = np.zeros(y.shape[1:], f32)
    for r in range(R):
        s = (s + y[r]).astype(f32)
        q = orc.fma32(y[r], y[r], q)
    mean = (s * (f32(1) / f32(R))).astype(f32)
    var = np.maximum(((q - (s * mean).astype(f32)).astype(f32) * (f32(1) / f32(R - 1))).astype(f32), f32(0))
    return (np.asarray(gamma, f32)[:, None, None] / np.sqrt((var + f32(EPS)).astype(f32))).astype(f32)


def vbn1_scale_welford(y, gamma):
    """The fp32 kernels' layer-1 scale with Welford's update in frame order: mean += d * (1 / n),
    m2 = fmaf(d, y - mean, m2), var = m2 / (R - 1)."""
    R = y.shape[0]
    mean = np.zeros(y.shape[1:], f32)
    m2 = np.zeros(y.shape[1:], f32)
    for r in range(R):
        d = (y[r] - mean).astype(f32)
        mean = orc.fma32(d, f32(1) / f32(r + 1), mean)
        m2 = orc.fma32(d, (y[r] - mean).astype(f32), m2)
    var = (m2 * (f32(1) / f32(R - 1))).astype(f32)
    return (np.asarray(gamma, f32)[:, None, None] / np.sqrt((var + f32(EPS)).astype(f32))).astype(f32)
