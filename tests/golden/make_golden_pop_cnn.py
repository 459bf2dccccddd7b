#!/usr/bin/env python
"""Generate the population-mode CNN golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden_pop_conv.py (make_golden's shims and ``run_reference`` driver): the policy is
``_cnn_oracle.policy_class`` -- an ``nn.Sequential`` of Conv2d / activation / Flatten / Linear layers built from
the packed ``dims`` of ``CNNSpec`` --, and the agent is ``tests/_pop_cnn_oracle.PixelPoint``, a point moved
smoothly by the outputs for 6 steps and rendered into 2x8x8 images, driven through the ``rollout(policy)`` that
``estorch_b200.PopulationAgent`` implements on top of ``rollout_population``.  To the reference they are just
another policy and agent.  The policies have 1,574 parameters, so the fixtures store theta0 and the table.
Writes only:

    es_pop_cnn_p16.npz      classic ES, P=16, sigma 0.05, 3 generations, ReLU hidden, Tanh output
    nsr_pop_cnn_p8.npz      NSR-ES, P=8, sigma 0.05, 4 generations, ELU hidden, identity output, 4-D BC (the
                            point after 3 and 6 steps)

    python tests/golden/make_golden_pop_cnn.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402  (installs the reference shims on import)
from _pop_cnn_oracle import DIMS, ES_POLICY, N_PARAMS, NSR_POLICY, PixelPoint, cnn_policy  # noqa: E402

TABLE_LEN = (N_PARAMS + 31) // 32 * 32 + 32 * 64


class PointRef(PixelPoint):
    """run_reference hands its agent obs / target / bc_obs / bc_dim keyword arguments; the point needs bc_dim."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        super().__init__(bc_dim=bc_dim)


def run(policy, cls, P, sigma, n_gen, table_seed, noise_seed, bc_dim=0):
    mg.MLP = cnn_policy(**policy)
    mg.SynthAgent = PointRef
    orc = mg.orc
    # run_reference sizes each noise row with orc.mlp_param_count(dims): give it the CNN's count
    mg.orc = types.SimpleNamespace(mlp_param_count=lambda d: N_PARAMS, noise_offsets=orc.noise_offsets)
    table = np.random.RandomState(table_seed).standard_normal(TABLE_LEN).astype(np.float16).astype(np.float32)
    try:
        out = mg.run_reference(cls, list(DIMS), P, sigma, n_gen, table, noise_seed, torch.zeros(1, 1),
                               torch.zeros(1, 2), bc_obs=1 if bc_dim else 0, bc_dim=bc_dim)
    finally:
        mg.orc = orc
    for k in ("obs", "target", "theta_before", "grad"):
        out.pop(k, None)
    out.update(hidden=policy["hidden"], out_tanh=policy["out_tanh"], n_conv=policy["n_conv"])
    return out


def main():
    out = run(ES_POLICY, mg.ref.ES, 16, 0.05, 3, table_seed=81, noise_seed=61)
    np.savez_compressed(os.path.join(HERE, "es_pop_cnn_p16.npz"), **out)
    out = run(NSR_POLICY, mg.ref.NSR_ES, 8, 0.05, 4, table_seed=82, noise_seed=67, bc_dim=4)
    np.savez_compressed(os.path.join(HERE, "nsr_pop_cnn_p8.npz"), **out)
    for f in ("es_pop_cnn_p16.npz", "nsr_pop_cnn_p8.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
