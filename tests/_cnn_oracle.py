"""TEST-ONLY: the convolutional evaluate (estk_eval_mlp with n_conv in bits 24-31, include/estk.h) in numpy -- an
fp32 forward and a float64 forward of a member's weights --, and ``policy_class`` builders for the test shapes.

A policy is described by its packed ``dims`` (``CNNSpec.dims``: ESTK_CNN_INPUT, one ESTK_CNN_CONV per conv, the
Linear widths) and its code (hidden | output | n_conv << 24), exactly what the library is handed."""
import numpy as np
import torch
from torch import nn


LOSS_XENT = 1 << 16
HIDDEN = {0: "relu", 1: "tanh", 3: "elu", 4: "silu", 5: "leaky_relu"}
_MODULES = {"relu": nn.ReLU, "tanh": nn.Tanh, "elu": nn.ELU, "silu": nn.SiLU, "leaky_relu": nn.LeakyReLU}


def unpack(dims, n_conv):
    """Packed dims -> ((c, h, w), [(out_c, k, stride, pad)], [linear widths])."""
    d = [int(x) & 0xffffffff for x in dims]
    shape = (d[0] & 1023, (d[0] >> 10) & 1023, (d[0] >> 20) & 1023)
    convs = [(f & 4095, (f >> 12) & 63, (f >> 18) & 63, (f >> 24) & 63) for f in d[1:1 + n_conv]]
    return shape, convs, d[1 + n_conv:]


def pack(shape, convs, linears):
    c, h, w = shape
    return (c | h << 10 | w << 20,) + tuple(o | k << 12 | s << 18 | p << 24 for o, k, s, p in convs) + tuple(linears)


def layer_shapes(shape, convs, linears):
    """[(w_shape, b_len)] of every layer in parameters_to_vector order, and the flattened width."""
    out, (c, h, w) = [], shape
    for o, k, s, p in convs:
        out.append(((o, c, k, k), o))
        c, h, w = o, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    fan = c * h * w
    for o in linears:
        out.append(((o, fan), o))
        fan = o
    return out, c * h * w


def param_count(dims, n_conv):
    shapes, _ = layer_shapes(*unpack(dims, n_conv))
    return sum(int(np.prod(ws)) + b for ws, b in shapes)


def _act(name, x):
    if name == "relu":
        return np.maximum(x, 0)
    if name == "tanh":
        return np.tanh(x)
    if name == "elu":
        return np.where(x > 0, x, np.expm1(np.minimum(x, 0)))
    if name == "silu":
        return x / (1 + np.exp(-x))
    return np.where(x > 0, x, x * x.dtype.type(0.01))


def _conv(x, wt, b, s, p, dt):
    """x [B, C, H, W], wt [O, C, k, k] -> [B, O, H', W'] in dtype dt (im2col, one matmul)."""
    B, C, H, W = x.shape
    O, _, k, _ = wt.shape
    xp = np.pad(x, ((0, 0), (0, 0), (p, p), (p, p)))
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    cols = np.empty((B, C, k, k, Ho, Wo), dt)
    for kh in range(k):
        for kw in range(k):
            cols[:, :, kh, kw] = xp[:, :, kh: kh + s * (Ho - 1) + 1: s, kw: kw + s * (Wo - 1) + 1: s]
    y = np.einsum("bkhw,ok->bohw", cols.reshape(B, C * k * k, Ho, Wo), wt.reshape(O, -1).astype(dt))
    return (y + b.astype(dt)[None, :, None, None]).astype(dt)


def forward(row, dims, code, obs, dt=np.float32):
    """One member's outputs [B, out] from its flat parameters ``row`` on ``obs`` [B, c, h, w], in dtype ``dt``
    (np.float32: the fp32 forward; np.float64: the float64 forward of the member's fp32 weights)."""
    n_conv = (int(code) >> 24) & 0xff
    shape, convs, linears = unpack(dims, n_conv)
    hidden, tanh_out = HIDDEN[int(code) & 0xff], bool(int(code) & 0x100)
    shapes, _ = layer_shapes(shape, convs, linears)
    row = np.asarray(row, np.float32).astype(dt)
    h, i = np.asarray(obs, np.float32).astype(dt), 0
    for li, (ws, bl) in enumerate(shapes):
        wt = row[i: i + int(np.prod(ws))].reshape(ws)
        i += wt.size
        b = row[i: i + bl]
        i += bl
        if li < n_conv:
            h = _act(hidden, _conv(h, wt, b, convs[li][2], convs[li][3], dt))
            if li == n_conv - 1:
                h = h.reshape(h.shape[0], -1)
        else:
            h = (h @ wt.T + b).astype(dt)
            if li + 1 < len(shapes):
                h = _act(hidden, h)
    return np.tanh(h) if tanh_out else h


def returns_of(y, target, xent, dt=np.float32):
    """Returns of outputs y [M, B, C]: the per-image value, then the sum over b in order, then -(S / count)."""
    y, tg = np.asarray(y).astype(dt), np.asarray(target, np.float32).astype(dt)
    if xent:
        m = y.max(-1, keepdims=True)
        lse = m[..., 0] + np.log(np.exp(y - m).sum(-1))
        per = lse * tg.sum(-1)[None] - (tg[None] * y).sum(-1)
    else:
        per = ((y - tg[None]) ** 2).sum(-1)
    S = np.zeros(y.shape[0], dt)
    for b in range(y.shape[1]):
        S = (S + per[:, b]).astype(dt)
    count = y.shape[1] * (1 if xent else y.shape[2])
    return (-(S / dt(count))).astype(dt)


def policy_class(n_conv, hidden="relu", out_tanh=False, form="sequential"):
    """A policy class built from ``dims`` (packed, as ``CNNSpec.dims``).  ``form``: "sequential" (an
    ``nn.Sequential`` with ``nn.Flatten``) or "custom" (a ``forward`` with ``.view`` and functional activations)."""
    fn = {"relu": torch.relu, "tanh": torch.tanh, "elu": nn.functional.elu, "silu": nn.functional.silu,
          "leaky_relu": nn.functional.leaky_relu}[hidden]

    class CNNPolicy(nn.Module):
        def __init__(self, dims):
            super().__init__()
            shape, convs, linears = unpack(dims, n_conv)
            c, mods, self.custom = shape[0], [], form == "custom"
            for o, k, s, p in convs:
                mods.append(nn.Conv2d(c, o, k, stride=s, padding=p))
                if not self.custom:
                    mods.append(_MODULES[hidden]())
                c = o
            _, fan = layer_shapes(shape, convs, linears)
            if not self.custom:
                mods.append(nn.Flatten())
            for li, o in enumerate(linears):
                mods.append(nn.Linear(fan, o))
                if not self.custom and li + 1 < len(linears):
                    mods.append(_MODULES[hidden]())
                fan = o
            if not self.custom and out_tanh:
                mods.append(nn.Tanh())
            self.net = nn.Sequential(*mods) if not self.custom else nn.ModuleList(mods)

        def forward(self, x):
            if not self.custom:
                return self.net(x)
            h = x
            layers = list(self.net)
            for i, m in enumerate(layers):
                if isinstance(m, nn.Linear) and h.dim() == 4:
                    h = h.view(h.shape[0], -1)
                h = m(h)
                if i + 1 < len(layers):
                    h = fn(h)
            return torch.tanh(h) if out_tanh else h
    return CNNPolicy


def image_task(B, shape=(1, 12, 12), n_classes=4, seed=0):
    """Seeded synthetic images: a bright blob in one of four quadrants on noise; one-hot quadrant targets."""
    g = torch.Generator().manual_seed(seed)
    c, h, w = shape
    x = 0.1 * torch.randn(B, c, h, w, generator=g)
    labels = torch.randint(0, n_classes, (B,), generator=g)
    for b in range(B):
        q = int(labels[b])
        r0, c0 = (q // 2) * (h // 2), (q % 2) * (w // 2)
        x[b, :, r0 + h // 8: r0 + h // 2 - h // 8, c0 + w // 8: c0 + w // 2 - w // 8] += 1.0
    return x, torch.nn.functional.one_hot(labels, n_classes).float()
