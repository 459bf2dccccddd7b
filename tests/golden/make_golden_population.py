#!/usr/bin/env python
"""Generate the population-agent golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden_act_ext.py (whose shims and ``run_reference`` driver this reuses): the agent
is ``tests/_pop_oracle.LinearWalker``, a deterministic damped linear system stepped for 40 steps, which
the reference drives through the ``rollout(policy)`` that ``estorch_b200.PopulationAgent`` implements on
top of ``rollout_population``.  The policy is a ReLU MLP with a Tanh output.  Writes only:

    es_pop_walker_p64.npz     classic ES, 24-64-64-4, P=64, sigma 0.05, 3 generations
    nsr_pop_walker_p32.npz    NSR-ES, 24-64-64-4, P=32, sigma 0.02, 5 generations, 48-D BC
                              (the walker's state after 20 and after 40 steps)

    python tests/golden/make_golden_population.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402  (installs the reference shims on import)
import make_golden_act_ext as mga  # noqa: E402
from _pop_oracle import LinearWalker  # noqa: E402


class WalkerRef(LinearWalker):
    """run_reference hands its agent obs / target / bc_obs / bc_dim keyword arguments; the walker needs none
    of the first three."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        super().__init__(bc_dim=bc_dim)


def main():
    mg.MLP = mga.mlp_class(torch.nn.ReLU, out_tanh=True)
    mg.SynthAgent = WalkerRef
    dims = [24, 64, 64, 4]
    none_obs, none_tgt = torch.zeros(1, 24), torch.zeros(1, 4)
    out = mg.run_reference(mg.ref.ES, dims, 64, 0.05, 3, mg.make_table(1 << 15, 61), 43, none_obs, none_tgt)
    np.savez_compressed(os.path.join(HERE, "es_pop_walker_p64.npz"), **out)
    out = mg.run_reference(mg.ref.NSR_ES, dims, 32, 0.02, 5, mg.make_table(1 << 15, 62), 47, none_obs, none_tgt,
                           bc_obs=1, bc_dim=48)
    np.savez_compressed(os.path.join(HERE, "nsr_pop_walker_p32.npz"), **out)
    for f in ("es_pop_walker_p64.npz", "nsr_pop_walker_p32.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
