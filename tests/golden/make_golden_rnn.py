#!/usr/bin/env python
"""Generate the recurrent-policy golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden_population.py (the shims and the ``run_reference`` driver of make_golden.py):
the agent is ``tests/_rnn_oracle.RecallAgent``, a deterministic cue-recall task, which the reference drives
through the ``rollout(policy)`` that ``estorch_b200.PopulationAgent`` implements on top of
``rollout_population`` (passing the recurrent state through the policy's ``forward(x, state)``).  The
policies are ``_rnn_oracle.policy_class``: one GRUCell / LSTMCell and a Linear head.  To the reference they
are just other policy classes.  Writes only:

    es_rnn_gru_p16.npz      classic ES, GRU 4-16-3 with a Tanh output, P=16, sigma 0.05, 3 generations
    nsr_rnn_lstm_p8.npz     NSR-ES, LSTM 4-8-3 with an identity output, P=8, sigma 0.02, 4 generations,
                            9-D BC (the last step's outputs for the three cues)

    python tests/golden/make_golden_rnn.py
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
from _rnn_oracle import RecallAgent, param_count, policy_class  # noqa: E402


class RecallRef(RecallAgent):
    """run_reference hands its agent obs / target / bc_obs / bc_dim keyword arguments; the task needs only
    bc_dim."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        super().__init__(bc_dim=bc_dim)


def run(cell, out_tanh, cls, dims, P, sigma, n_gen, table, noise_seed, **kw):
    mg.MLP = policy_class(cell, out_tanh)
    # run_reference sizes each noise row with orc.mlp_param_count(dims): give it the recurrent policy's count
    orc = mg.orc
    mg.orc = types.SimpleNamespace(mlp_param_count=lambda d: param_count(cell, d), noise_offsets=orc.noise_offsets)
    try:
        none_obs, none_tgt = torch.zeros(1, 4), torch.zeros(1, 3)
        return mg.run_reference(cls, list(dims), P, sigma, n_gen, table, noise_seed, none_obs, none_tgt, **kw)
    finally:
        mg.orc = orc


def main():
    mg.SynthAgent = RecallRef
    out = run("gru", True, mg.ref.ES, (4, 16, 3), 16, 0.05, 3, mg.make_table(1 << 14, 71), 53)
    np.savez_compressed(os.path.join(HERE, "es_rnn_gru_p16.npz"), **out)
    out = run("lstm", False, mg.ref.NSR_ES, (4, 8, 3), 8, 0.02, 4, mg.make_table(1 << 14, 72), 59,
              bc_obs=1, bc_dim=9)
    np.savez_compressed(os.path.join(HERE, "nsr_rnn_lstm_p8.npz"), **out)
    for f in ("es_rnn_gru_p16.npz", "nsr_rnn_lstm_p8.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
