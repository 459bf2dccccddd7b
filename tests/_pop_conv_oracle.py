"""TEST-ONLY: the action mode of estk_eval_conv_vbn (ESTK_ACTIONS) in numpy, an oracle stand-in backend that
serves it, the Atari-example policy, and the deterministic pixel agent of the conv population tests and goldens.

The oracle folds the VirtualBatchNorm statistics as the kernels do (a = gamma / sqrt(var + 1e-5),
c = beta - mean * a, per (C, H, W) position; mean and unbiased var over the reference batch, estorch/
modules.py:48-58) and runs the convolutions as fp32 matrix products, so it agrees with the kernels to fp32
accumulation order, not bit for bit."""
import numpy as np
import torch
from numpy.lib.stride_tricks import sliding_window_view

from oracle import es_oracle as orc
from _oracle_backend import _np
from _pop_oracle import PopOracleBackend
from estorch_b200 import PopulationAgent, VirtualBatchNorm

STATS_FLOATS = 17984        # include/estk.h ESTK_CONV_VBN_STATS_FLOATS
P1, P2 = 16 * 20 * 20, 32 * 9 * 9
f32 = np.float32


class AtariPolicy(torch.nn.Module):
    """The conv + VirtualBatchNorm policy of the reference's Atari example (examples/atari.py:14-37), with
    this package's VirtualBatchNorm; the parameters register in the same order."""

    def __init__(self, n_actions, xref):
        super().__init__()
        self.xref = xref
        self.conv1 = torch.nn.Conv2d(4, 16, 8, 4)
        self.bn1 = VirtualBatchNorm(16)
        self.conv2 = torch.nn.Conv2d(16, 32, 4, 2)
        self.bn2 = VirtualBatchNorm(32)
        self.fc1 = torch.nn.Linear(2592, 256)
        self.fc2 = torch.nn.Linear(256, n_actions)

    def forward(self, x):
        F = torch.nn.functional
        xref = F.relu(self.bn1(self.conv1(self.xref)))
        F.relu(self.bn2(self.conv2(xref)))
        x = F.relu(self.bn1(self.conv1(x)))
        x = F.relu(self.bn2(self.conv2(x)))
        x = F.relu(self.fc1(x.view(-1, 2592)))
        return self.fc2(x)


def unflatten(row, n_actions):
    p, idx = {}, 0
    for name, shape in orc.atari_param_layout(n_actions):
        sz = int(np.prod(shape))
        p[name] = row[idx:idx + sz].reshape(shape).astype(f32)
        idx += sz
    return p


def _conv(x, w, b, stride):
    """x [M, N, C, H, W] (member m's images), w [M, O, C, k, k], b [M, O] -> [M, N, O, OH, OW] in fp32."""
    M, N, C, H, W = x.shape
    k = w.shape[-1]
    v = sliding_window_view(x, (k, k), axis=(3, 4))[:, :, :, ::stride, ::stride]     # [M,N,C,OH,OW,k,k]
    OH, OW = v.shape[3], v.shape[4]
    cols = v.transpose(0, 1, 3, 4, 2, 5, 6).reshape(M, N * OH * OW, C * k * k)
    y = np.matmul(cols, w.reshape(M, w.shape[1], -1).transpose(0, 2, 1)) + b[:, None, :]
    return y.reshape(M, N, OH, OW, -1).transpose(0, 1, 4, 2, 3).astype(f32)


def _params(rows, n_actions):
    ps = [unflatten(r, n_actions) for r in np.asarray(rows, dtype=f32)]
    return {k: np.stack([p[k] for p in ps]) for k in ps[0]}


def conv_stats(rows, n_actions, xref):
    """rows [M, n], xref [R, 4, 84, 84] -> [M, STATS_FLOATS]: a1, c1 [16*20*20], a2, c2 [32*9*9] per member."""
    p = _params(rows, n_actions)
    M = p["conv1.w"].shape[0]
    x = np.broadcast_to(np.asarray(xref, dtype=f32)[None], (M,) + tuple(xref.shape))

    def fold(y, g, b):
        mean = y.mean(axis=1, dtype=f32)
        var = y.var(axis=1, ddof=1, dtype=f32)
        a = (g[:, :, None, None] / np.sqrt(var + f32(1e-5))).astype(f32)
        return a, (b[:, :, None, None] - mean * a).astype(f32)

    r1 = _conv(x, p["conv1.w"], p["conv1.b"], 4)
    a1, c1 = fold(r1, p["bn1.w"], p["bn1.b"])
    h = np.maximum(r1 * a1[:, None] + c1[:, None], 0).astype(f32)
    r2 = _conv(h, p["conv2.w"], p["conv2.b"], 2)
    a2, c2 = fold(r2, p["bn2.w"], p["bn2.b"])
    return np.concatenate([a1.reshape(M, -1), c1.reshape(M, -1), a2.reshape(M, -1), c2.reshape(M, -1)], 1)


def conv_act(rows, n_actions, stats, obs):
    """rows [M, n], stats [M, STATS_FLOATS], obs [M, B, 4, 84, 84] -> outputs [M, B, A] (fp32)."""
    p = _params(rows, n_actions)
    st = np.asarray(stats, dtype=f32)
    M = st.shape[0]
    a1, c1 = st[:, :P1].reshape(M, 1, 16, 20, 20), st[:, P1:2 * P1].reshape(M, 1, 16, 20, 20)
    a2, c2 = st[:, 2 * P1:2 * P1 + P2].reshape(M, 1, 32, 9, 9), st[:, 2 * P1 + P2:].reshape(M, 1, 32, 9, 9)
    h = np.maximum(_conv(np.asarray(obs, dtype=f32), p["conv1.w"], p["conv1.b"], 4) * a1 + c1, 0).astype(f32)
    h = np.maximum(_conv(h, p["conv2.w"], p["conv2.b"], 2) * a2 + c2, 0).astype(f32)
    h = h.reshape(M, h.shape[1], 2592)
    h = np.maximum(np.matmul(h, p["fc1.w"].transpose(0, 2, 1)) + p["fc1.b"][:, None], 0).astype(f32)
    return (np.matmul(h, p["fc2.w"].transpose(0, 2, 1)) + p["fc2.b"][:, None]).astype(f32)


class PopConvOracleBackend(PopOracleBackend):
    """PopOracleBackend plus ``act_conv_vbn`` (CudaBackend's signature); counts its stats and act launches."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.stats_calls = 0
        self.conv_act_calls = 0

    def act_conv_vbn(self, n_actions, theta, table, offsets, order, pairs, sigma, xref, obs, out, stats,
                     table16=None):
        if offsets is None:
            rows = _np(theta)[None, :]
        else:
            if table16 is not None:
                assert table16.dtype == torch.float16
                table = table16.float()
            rows, _ = orc.sample_population(_np(theta), _np(table), _np(offsets), sigma)
        assert tuple(stats.shape) == (rows.shape[0], STATS_FLOATS)
        if xref is not None:
            self.stats_calls += 1
            stats.copy_(torch.from_numpy(conv_stats(rows, int(n_actions), _np(xref))))
        if obs is not None:
            self.conv_act_calls += 1
            assert tuple(obs.shape) == (rows.shape[0], obs.shape[1], 4, 84, 84)
            assert tuple(out.shape) == (rows.shape[0], obs.shape[1], int(n_actions))
            out.copy_(torch.from_numpy(conv_act(rows, int(n_actions), _np(stats), _np(obs))))


class PixelWalker(PopulationAgent):
    """A point in the plane rendered into 84x84 frames: channel i is a Gaussian blob of width w_i around the
    point (the four widths stand in for a frame stack).  The four logits move it smoothly,
    s' = s + 0.1 * tanh(GAIN * (y0 - y1, y2 - y3)), no argmax, so fp32 order differences in the forward stay in
    the last bits of the returns; reward -|s' - goal|^2 per step, fixed start and horizon.  Vectorised over
    members.  ``bc_dim`` = 4 makes it an NS-family agent: the point at the middle and at the end."""

    WIDTHS = (0.08, 0.12, 0.18, 0.27)
    GAIN = 0.005        # the logits of an untrained conv policy reach the hundreds

    def __init__(self, horizon=8, bc_dim=0):
        assert bc_dim in (0, 4)
        self.horizon, self.bc_dim = horizon, bc_dim
        self.s0 = torch.tensor([-0.5, 0.35])
        self.goal = torch.tensor([0.4, -0.25])

    def frames(self, s):
        """[M, 2] points -> [M, 4, 84, 84] float32 frames."""
        g = (torch.arange(84, device=s.device, dtype=torch.float32) + 0.5) / 42.0 - 1.0
        d2 = (g[None, :, None] - s[:, 0, None, None]) ** 2 + (g[None, None, :] - s[:, 1, None, None]) ** 2
        w = torch.tensor(self.WIDTHS, device=s.device, dtype=torch.float32)
        return (torch.exp(-d2[:, None] / (2 * w * w)[None, :, None, None]) + self.background(s.device)).contiguous()

    @staticmethod
    def background(device):
        """A fixed texture of amplitude 0.5 behind the blobs, so the frames look like the reference batch's."""
        return (0.5 * torch.rand(1, 4, 84, 84, generator=torch.Generator().manual_seed(5))).to(device)

    def rollout_population(self, act, members):
        dev = self.device
        s = self.s0.to(dev).expand(members, 2).contiguous()
        goal = self.goal.to(dev)
        ret = torch.zeros(members, device=dev)
        mid = s
        for t in range(self.horizon):
            y = act(self.frames(s))
            s = s + 0.1 * torch.tanh(self.GAIN * torch.stack([y[:, 0] - y[:, 1], y[:, 2] - y[:, 3]], 1))
            ret = ret - ((s - goal) ** 2).sum(1)
            if t + 1 == self.horizon // 2:
                mid = s
        if self.bc_dim:
            return ret, torch.cat([mid, s], 1)
        return ret


def walker_xref(R=4, seed=11):
    """R reference frames of the walker at points of a random walk (random actions, as the reference collects
    its Atari reference batch, examples/atari.py:89-120), over a uniform background of amplitude 0.5 so that
    every pixel varies over the batch: VBN over a nearly constant pixel scales it by up to 1/sqrt(1e-5), and
    the forward would then magnify fp32 rounding far beyond the tests' bars."""
    g = torch.Generator().manual_seed(seed)
    s = torch.zeros(1, 2)
    frames = []
    ag = PixelWalker()
    for _ in range(R):
        s = (s + 0.25 * torch.randn(1, 2, generator=g)).clamp(-0.9, 0.9)
        frames.append(ag.frames(s) - ag.background(s.device) + 0.5 * torch.rand(1, 4, 84, 84, generator=g))
    return torch.cat(frames).contiguous()


# ---------------------------------------------------------------- golden fixtures: regenerable inputs
def golden_theta0(n_actions, seed):
    """A deterministic starting point for the goldens, regenerated instead of stored (680 k parameters):
    conv / linear weights and biases uniform in +-1/sqrt(fan_in) (torch's default bound), VBN gamma
    1 + 0.1 N(0,1), beta 0.1 N(0,1)."""
    rs = np.random.RandomState(seed)
    parts = []
    for name, shape in orc.atari_param_layout(n_actions):
        if name.startswith("bn"):
            base = 1.0 if name.endswith(".w") else 0.0
            parts.append(base + 0.1 * rs.standard_normal(shape))
        else:
            fan_in = {"conv1": 256, "conv2": 256, "fc1": 2592, "fc2": 256}[name.split(".")[0]]
            parts.append(rs.uniform(-1, 1, shape) / np.sqrt(fan_in))
    return np.concatenate([p.reshape(-1) for p in parts]).astype(f32)


def golden_table(length, seed):
    """Unit normals rounded to fp16-representable values (like estk_fill_noise_table), regenerated."""
    return np.random.RandomState(seed).standard_normal(length).astype(np.float16).astype(f32)


def theta_subset(n):
    """Indices of theta a golden stores: every conv / VBN parameter, every 64th fc1 weight, fc1.b, fc2."""
    return np.concatenate([np.arange(12432), np.arange(12432, 12432 + 663552, 64), np.arange(12432 + 663552, n)])
