#!/usr/bin/env python
"""Generate the conv population-agent golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden_population.py (make_golden's shims and ``run_reference`` driver): the policy is
the reference's own Atari ``Policy`` (examples/atari.py:14-37, conv + VirtualBatchNorm) with 4 actions and
a reference batch of R = 8 frames (over 4 frames the per-position VBN variances are so noisy that a few
positions scale their input by hundreds, and fp32 order differences no longer stay within the bars), and the agent is ``tests/_pop_conv_oracle.PixelWalker``, a point moved
smoothly by the logits for 8 steps and rendered into 84x84 frames, driven through the ``rollout(policy)``
that ``estorch_b200.PopulationAgent`` implements on top of ``rollout_population``.

The network has 677,268 parameters, so the inputs are regenerated from seeds rather than stored: the noise
table (``golden_table``), the starting parameters (``golden_theta0``, written into the reference policy
after its own initialisation) and the reference frames (``walker_xref``).  Of ES's theta after training and
of its best theta the fixture keeps the ``theta_subset`` entries.  Writes only:

    es_pop_conv_p16.npz     classic ES, P=16, sigma 0.05, 3 generations
    nsr_pop_conv_p8.npz     NSR-ES, P=8, sigma 0.05, 4 generations, 4-D BC (the point after 4 and 8 steps)

    python tests/golden/make_golden_pop_conv.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402  (installs the reference shims on import)
import atari as ref_atari  # noqa: E402  (the reference example module, gym / skimage shimmed)
from _pop_conv_oracle import PixelWalker, golden_table, golden_theta0, theta_subset, walker_xref  # noqa: E402

A, R = 4, 8
N = 12432 + 256 * 2592 + 256 + 256 * A + A
TABLE_LEN, XREF_SEED = (N + 31) // 32 * 32 + 32 * 256, 11


class WalkerRef(PixelWalker):
    """run_reference hands its agent obs / target / bc_obs / bc_dim keyword arguments; the walker needs bc_dim."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        super().__init__(bc_dim=bc_dim)


def policy_class(seed0):
    """The reference Policy, its parameters then set to golden_theta0(A, seed0 + k) for its k-th instance."""
    count = [0]

    class RefPolicy(ref_atari.Policy):
        def __init__(self, dims):
            super().__init__(A, walker_xref(R, XREF_SEED))
            torch.nn.utils.vector_to_parameters(torch.from_numpy(golden_theta0(A, seed0 + count[0])),
                                                self.parameters())
            count[0] += 1
    return RefPolicy, count


def seed_of(flat, seed0, count):
    for k in range(count):
        if np.array_equal(flat, golden_theta0(A, seed0 + k)):
            return seed0 + k
    raise AssertionError("a starting theta that is no golden_theta0")


def run(cls, P, sigma, n_gen, table_seed, noise_seed, seed0, bc_dim=0):
    mg.MLP, count = policy_class(seed0)
    mg.SynthAgent = WalkerRef
    mlp_param_count = mg.orc.mlp_param_count
    mg.orc.mlp_param_count = lambda dims: N        # run_reference sizes the noise rows by the policy's n
    try:
        out = mg.run_reference(cls, [A], P, sigma, n_gen, golden_table(TABLE_LEN, table_seed), noise_seed,
                               torch.zeros(1, 1), torch.zeros(1, A), bc_obs=1 if bc_dim else 0, bc_dim=bc_dim)
    finally:
        mg.orc.mlp_param_count = mlp_param_count
    sub = theta_subset(N)
    keep = dict(P=P, sigma=sigma, noise_seed=noise_seed, table_seed=table_seed, table_len=TABLE_LEN, R=R,
                xref_seed=XREF_SEED, n_actions=A, theta_subset_after=out["theta_after"][-1][sub],
                **{k: out[k] for k in ("offsets", "returns", "episode_reward", "best_reward", "idx", "archive_len")})
    if "meta_theta0" in out:
        keep["meta_seeds"] = np.array([seed_of(f, seed0, count[0]) for f in out["meta_theta0"]])
        keep["archive0"], keep["archive_final"], keep["k"] = out["archive0"], out["archive_final"], out["k"]
    else:
        keep["theta0_seed"] = seed_of(out["theta0"], seed0, count[0])
        keep["best_theta_subset"] = out["best_theta"][sub]
    return keep


def main():
    out = run(mg.ref.ES, 16, 0.05, 3, table_seed=71, noise_seed=53, seed0=100)
    np.savez_compressed(os.path.join(HERE, "es_pop_conv_p16.npz"), **out)
    out = run(mg.ref.NSR_ES, 8, 0.05, 4, table_seed=72, noise_seed=57, seed0=200, bc_dim=4)
    np.savez_compressed(os.path.join(HERE, "nsr_pop_conv_p8.npz"), **out)
    for f in ("es_pop_conv_p16.npz", "nsr_pop_conv_p8.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
