#!/usr/bin/env python
"""Generate the cross-entropy golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden.py (whose shims and ``run_reference`` driver this reuses):
the reference classes run an agent whose rollout returns minus the soft-target
cross-entropy of the policy's logits -- to the reference it is just another agent class.
Writes only the two fixtures below, so the existing ones are not rewritten:

    es_xent_p64.npz    classic ES, 4-64-64-3 ReLU MLP, one-hot targets, P=64, 3 generations
    nsr_xent_p32.npz   NSR-ES, 24-64-64-4 ReLU MLP, soft targets, P=32, 5 generations, 256-D BC

    python tests/golden/make_golden_xent.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (installs the reference shims on import)


class XentAgent:
    """rollout = mean_b sum_c target_bc * log_softmax(policy(obs))_bc; NS: + bc = the logits
    policy(obs[:bc_obs]).flatten()[:bc_dim]."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        self.obs, self.target, self.bc_obs, self.bc_dim = obs, target, bc_obs, bc_dim

    def rollout(self, policy):
        with torch.no_grad():
            out = policy(self.obs)
            r = float((self.target * torch.log_softmax(out, 1)).sum(1).mean())
            if self.bc_dim:
                return r, out[:self.bc_obs].flatten()[:self.bc_dim].numpy().copy()
        return r


def main():
    g = torch.Generator().manual_seed(8765)
    mg.SynthAgent = XentAgent                          # the agent class run_reference hands the reference
    # --- classic ES, 3 classes, one-hot targets, P=64 ---
    dims = [4, 64, 64, 3]
    obs = torch.randn(256, 4, generator=g)
    labels = torch.randint(0, 3, (256,), generator=g)
    tgt = torch.nn.functional.one_hot(labels, 3).to(torch.float32)
    out = mg.run_reference(mg.ref.ES, dims, 64, 0.1, 3, mg.make_table(1 << 15, 47), 23, obs, tgt)
    np.savez_compressed(os.path.join(HERE, "es_xent_p64.npz"), **out)

    # --- NSR-ES, 4 classes, soft targets (rows sum to 1), P=32 ---
    dims = [24, 64, 64, 4]
    obs = torch.randn(256, 24, generator=g)
    tgt = torch.softmax(2.0 * torch.randn(256, 4, generator=g), 1)
    out = mg.run_reference(mg.ref.NSR_ES, dims, 32, 0.02, 5, mg.make_table(1 << 15, 48), 29, obs, tgt,
                           bc_obs=64, bc_dim=256)
    np.savez_compressed(os.path.join(HERE, "nsr_xent_p32.npz"), **out)
    for f in ("es_xent_p64.npz", "nsr_xent_p32.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
