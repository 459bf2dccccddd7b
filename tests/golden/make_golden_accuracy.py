#!/usr/bin/env python
"""Generate the classification-accuracy golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden.py (whose shims and ``run_reference`` driver this reuses): the
reference classes run an agent whose rollout returns the fraction of the batch whose logits'
argmax is the target's argmax -- to the reference it is just another agent class.  Writes only
the two fixtures below, so the existing ones are not rewritten:

    es_accuracy_p64.npz    classic ES, 8-64-64-4 ReLU MLP, one-hot targets, B=200, P=64, 3 generations
    nsr_accuracy_p32.npz   NSR-ES, 16-64-64-5 ReLU MLP, soft targets, B=256, P=32, 4 generations, 160-D BC

Accuracy returns are multiples of 1/B and tie often; the reference ranks them with an unstable argsort,
so only the per-generation returns (a function of theta_before, the offsets and the batch) are compared
bit for bit by the tests, not the updates.

    python tests/golden/make_golden_accuracy.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (installs the reference shims on import)


class AccuracyAgent:
    """rollout = mean_b [argmax policy(obs)_b == argmax target_b] (an exact count over B, one fp32 divide);
    NS: + bc = the logits policy(obs[:bc_obs]).flatten()[:bc_dim]."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        self.obs, self.target, self.bc_obs, self.bc_dim = obs, target, bc_obs, bc_dim

    def rollout(self, policy):
        with torch.no_grad():
            out = policy(self.obs)
            r = float((out.argmax(1) == self.target.argmax(1)).float().mean())
            if self.bc_dim:
                return r, out[:self.bc_obs].flatten()[:self.bc_dim].numpy().copy()
        return r


def _task(g, B, d, C):
    """Inputs whose class is a noisy linear function of them, so that accuracy has room to move."""
    obs = torch.randn(B, d, generator=g)
    w = torch.randn(d, C, generator=g)
    labels = (obs @ w + 0.5 * torch.randn(B, C, generator=g)).argmax(1)
    return obs, labels


def main():
    g = torch.Generator().manual_seed(9182)
    mg.SynthAgent = AccuracyAgent                      # the agent class run_reference hands the reference
    # --- classic ES, 4 classes, one-hot targets, B=200, P=64 ---
    dims = [8, 64, 64, 4]
    obs, labels = _task(g, 200, 8, 4)
    tgt = torch.nn.functional.one_hot(labels, 4).to(torch.float32)
    out = mg.run_reference(mg.ref.ES, dims, 64, 0.1, 3, mg.make_table(1 << 15, 61), 31, obs, tgt)
    np.savez_compressed(os.path.join(HERE, "es_accuracy_p64.npz"), **out)

    # --- NSR-ES, 5 classes, soft targets (the label is each row's largest weight), P=32 ---
    dims = [16, 64, 64, 5]
    obs, labels = _task(g, 256, 16, 5)
    tgt = torch.softmax(torch.randn(256, 5, generator=g) + 3.0 * torch.nn.functional.one_hot(labels, 5), 1)
    out = mg.run_reference(mg.ref.NSR_ES, dims, 32, 0.05, 4, mg.make_table(1 << 15, 62), 37, obs, tgt,
                           bc_obs=32, bc_dim=160)
    np.savez_compressed(os.path.join(HERE, "nsr_accuracy_p32.npz"), **out)
    for f in ("es_accuracy_p64.npz", "nsr_accuracy_p32.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
