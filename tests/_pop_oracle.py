"""TEST-ONLY: the act-mode forward of estk_eval_mlp with ESTK_ACTIONS in numpy, an oracle stand-in backend
that serves it, and the deterministic population agents of the population-mode tests and goldens.

Rounding model of the act-mode kernel (estorch_b200/csrc/estk_eval_mlp_act.cu): W = theta +- (sigma*t)
with the reference's two fp32 roundings; per output one fma chain from 0 in ascending k; + bias in fp32;
the hidden activation of ``_act_ext_oracle.HIDDEN``; tanh in fp32 for the Tanh output.  The fp32 fma is
emulated in fp64: the product of two fp32 values is exact there, the sum is rounded to fp64 and then to
fp32 (a double rounding that differs from one fma rounding only in rare ties)."""
import numpy as np
import torch

from oracle import es_oracle as orc
from _act_ext_oracle import ActExtOracleBackend, HIDDEN_CODES, HIDDEN
from _oracle_backend import _np
from estorch_b200 import PopulationAgent

ACTIONS = 3 << 16        # include/estk.h ESTK_ACTIONS
OUT_TANH = 1 << 8


def act_forward(rows, dims, obs, code):
    """rows [M, n] (each member's parameters), obs [M, B, in] -> outputs [M, B, out] (fp32)."""
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
        h = HIDDEN[hidden](y).astype(np.float32) if li + 1 < n_layers else y
    return np.tanh(h).astype(np.float32) if code & OUT_TANH else h


class PopOracleBackend(ActExtOracleBackend):
    """ActExtOracleBackend plus ``act_mlp`` (CudaBackend's signature); counts its calls in ``act_calls``."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.act_calls = 0

    def act_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, out, act=0, table16=None):
        self.act_calls += 1
        dims = [int(d) for d in dims]
        if offsets is None:
            rows = _np(theta)[None, :]
        else:
            if table16 is not None:
                assert table16.dtype == torch.float16
                if table is not None:
                    assert np.array_equal(_np(table16).astype(np.float32), _np(table))
                table = table16.float()
            rows, _ = orc.sample_population(_np(theta), _np(table), _np(offsets), sigma)
        assert tuple(obs.shape) == (rows.shape[0], obs.shape[1], dims[0]) == tuple(out.shape[:2]) + (dims[0],)
        out.copy_(torch.from_numpy(act_forward(rows, dims, _np(obs), (act & 0xffff) | ACTIONS)))


class LinearWalker(PopulationAgent):
    """A damped linear system with 24 state and 4 action dimensions, a fixed reset state and a fixed horizon:
    s' = A s + Bm a; reward -mean(s'^2) - 0.01 mean(a^2) per step.  Deterministic and
    vectorised over members.  ``bc_dim`` > 0 makes it an NS-family agent: the behaviour characteristic is
    the state at the middle and at the end of the episode."""

    def __init__(self, horizon=40, bc_dim=0):
        g = torch.Generator().manual_seed(2024)
        q, _ = torch.linalg.qr(torch.randn(24, 24, generator=g, dtype=torch.float64))
        self.A = (0.9 * q).to(torch.float32)
        self.Bm = (0.3 * torch.randn(24, 4, generator=g)).to(torch.float32)
        self.s0 = torch.randn(24, generator=g).to(torch.float32)
        self.horizon = horizon
        self.bc_dim = bc_dim
        assert bc_dim in (0, 48)

    def rollout_population(self, act, members):
        dev = self.device
        A, Bm = self.A.to(dev), self.Bm.to(dev)
        s = self.s0.to(dev).expand(members, 24).contiguous()
        ret = torch.zeros(members, device=dev)
        mid = None
        for t in range(self.horizon):
            a = act(s)
            s = s @ A.T + a @ Bm.T
            ret = ret - (s * s).mean(1) - 0.01 * (a * a).mean(1)
            if t + 1 == self.horizon // 2:
                mid = s
        if self.bc_dim:
            return ret, torch.cat([mid, s], 1)
        return ret
