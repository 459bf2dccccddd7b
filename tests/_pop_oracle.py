"""TEST-ONLY: the deterministic population agent of the population-mode tests and goldens."""
import torch

from estorch_b200 import PopulationAgent


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
