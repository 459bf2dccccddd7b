#!/usr/bin/env python
"""Generate the Tanh-policy golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden.py (whose shims and ``run_reference`` driver this reuses):
the reference classes run a policy whose hidden activations are ``nn.Tanh`` -- to the
reference it is just another policy class.  Writes only the two fixtures below, so the
existing ones are not rewritten:

    es_tanh_cartpole_p64.npz   classic ES, 4-64-64-2, Tanh hidden, identity output, P=64, 3 generations
    nsr_tanh_bipedal_p32.npz   NSR-ES, 24-64-64-4, Tanh hidden + Tanh output, P=32, 5 generations, 256-D BC

    python tests/golden/make_golden_tanh.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (installs the reference shims on import)


class TanhMLP(torch.nn.Module):
    """Linear -> Tanh -> ... -> Linear [-> Tanh]."""
    OUT_TANH = False

    def __init__(self, dims):
        super().__init__()
        layers = []
        for i in range(len(dims) - 1):
            layers.append(torch.nn.Linear(dims[i], dims[i + 1]))
            if i + 2 < len(dims) or self.OUT_TANH:
                layers.append(torch.nn.Tanh())
        self.net = torch.nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


class TanhTanhMLP(TanhMLP):
    OUT_TANH = True


def main():
    g = torch.Generator().manual_seed(4321)
    # --- classic ES, CartPole-shape Tanh MLP, P=64 ---
    dims = [4, 64, 64, 2]
    obs = torch.randn(256, 4, generator=g)
    tgt = torch.randn(256, 2, generator=g)
    mg.MLP = TanhMLP                                   # the policy class run_reference hands the reference
    out = mg.run_reference(mg.ref.ES, dims, 64, 0.1, 3, mg.make_table(1 << 15, 45), 17, obs, tgt)
    np.savez_compressed(os.path.join(HERE, "es_tanh_cartpole_p64.npz"), **out)

    # --- NSR-ES, BipedalWalker-shape Tanh MLP with a Tanh output, P=32; targets within (-1, 1) ---
    dims = [24, 64, 64, 4]
    obs = torch.randn(256, 24, generator=g)
    tgt = torch.rand(256, 4, generator=g) * 1.8 - 0.9
    mg.MLP = TanhTanhMLP
    out = mg.run_reference(mg.ref.NSR_ES, dims, 32, 0.02, 5, mg.make_table(1 << 15, 46), 19, obs, tgt,
                           bc_obs=64, bc_dim=256)
    np.savez_compressed(os.path.join(HERE, "nsr_tanh_bipedal_p32.npz"), **out)
    for f in ("es_tanh_cartpole_p64.npz", "nsr_tanh_bipedal_p32.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
