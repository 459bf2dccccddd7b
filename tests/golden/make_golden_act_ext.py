#!/usr/bin/env python
"""Generate the ELU / SiLU / LeakyReLU golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden_tanh.py and make_golden_xent.py (whose shims, ``run_reference``
driver and cross-entropy agent this reuses): to the reference the policies are just other policy
classes.  Writes only the three fixtures below, so the existing ones are not rewritten:

    es_elu_cartpole_p64.npz     classic ES, 4-64-64-2, ELU hidden, identity output, P=64, 3 generations
    nsr_silu_bipedal_p32.npz    NSR-ES, 24-64-64-4, SiLU hidden + Tanh output, P=32, 5 generations, 256-D BC
    es_leaky_xent_p64.npz       classic ES, 4-64-64-3, LeakyReLU hidden, cross-entropy on one-hot targets,
                                P=64, 3 generations

    python tests/golden/make_golden_act_ext.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (installs the reference shims on import)
import make_golden_xent as mgx  # noqa: E402


def mlp_class(act, out_tanh=False):
    class ActMLP(torch.nn.Module):
        """Linear -> act -> ... -> Linear [-> Tanh]."""
        def __init__(self, dims):
            super().__init__()
            layers = []
            for i in range(len(dims) - 1):
                layers.append(torch.nn.Linear(dims[i], dims[i + 1]))
                if i + 2 < len(dims):
                    layers.append(act())
            if out_tanh:
                layers.append(torch.nn.Tanh())
            self.net = torch.nn.Sequential(*layers)

        def forward(self, x):
            return self.net(x)
    return ActMLP


def main():
    g = torch.Generator().manual_seed(9876)
    synth = mg.SynthAgent
    # --- classic ES, CartPole-shape ELU MLP, P=64 ---
    dims = [4, 64, 64, 2]
    obs = torch.randn(256, 4, generator=g)
    tgt = torch.randn(256, 2, generator=g)
    mg.MLP = mlp_class(torch.nn.ELU)                  # the policy class run_reference hands the reference
    out = mg.run_reference(mg.ref.ES, dims, 64, 0.1, 3, mg.make_table(1 << 15, 51), 31, obs, tgt)
    np.savez_compressed(os.path.join(HERE, "es_elu_cartpole_p64.npz"), **out)

    # --- NSR-ES, BipedalWalker-shape SiLU MLP with a Tanh output, P=32; targets within (-1, 1) ---
    dims = [24, 64, 64, 4]
    obs = torch.randn(256, 24, generator=g)
    tgt = torch.rand(256, 4, generator=g) * 1.8 - 0.9
    mg.MLP = mlp_class(torch.nn.SiLU, out_tanh=True)
    out = mg.run_reference(mg.ref.NSR_ES, dims, 32, 0.02, 5, mg.make_table(1 << 15, 52), 37, obs, tgt,
                           bc_obs=64, bc_dim=256)
    np.savez_compressed(os.path.join(HERE, "nsr_silu_bipedal_p32.npz"), **out)

    # --- classic ES, LeakyReLU MLP, cross-entropy on one-hot targets over 3 classes, P=64 ---
    dims = [4, 64, 64, 3]
    obs = torch.randn(256, 4, generator=g)
    labels = torch.randint(0, 3, (256,), generator=g)
    tgt = torch.nn.functional.one_hot(labels, 3).to(torch.float32)
    mg.MLP = mlp_class(torch.nn.LeakyReLU)
    mg.SynthAgent = mgx.XentAgent
    out = mg.run_reference(mg.ref.ES, dims, 64, 0.1, 3, mg.make_table(1 << 15, 53), 41, obs, tgt)
    mg.SynthAgent = synth
    np.savez_compressed(os.path.join(HERE, "es_leaky_xent_p64.npz"), **out)
    for f in ("es_elu_cartpole_p64.npz", "nsr_silu_bipedal_p32.npz", "es_leaky_xent_p64.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
