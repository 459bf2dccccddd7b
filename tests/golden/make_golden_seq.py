#!/usr/bin/env python
"""Generate the recurrent sequence-evaluate golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden_rnn.py (the shims and the ``run_reference`` driver of make_golden.py): the agent is
``estorch_b200.SequenceAgent``, whose ``rollout(policy)`` runs the policy over every sequence with plain torch,
passing the recurrent state through ``forward(x, state)``.  The policies are ``_rnn_oracle.policy_class``: one
GRUCell / LSTMCell and a Linear head.  To the reference they are just another policy and agent.  Writes only:

    es_seq_gru_p16.npz      classic ES, GRU 3-16-2 with a Tanh output, squared error over B=4 sequences of
                            T=5 steps of random regression data, P=16, sigma 0.05, 3 generations
    nsr_seq_lstm_p8.npz     NSR-ES, LSTM 4-8-3 with an identity output, cross-entropy on the delayed-recall
                            dataset (only the last step is scored), P=8, sigma 0.02, 4 generations,
                            54-D BC (every output of the 3 sequences, (b, t, c) order)

    python tests/golden/make_golden_seq.py
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
from _rnn_oracle import param_count, policy_class  # noqa: E402
from _seq_oracle import recall_dataset  # noqa: E402
from estorch_b200 import SequenceAgent  # noqa: E402


class SequenceXent(SequenceAgent):
    """run_reference hands its agent obs / target / bc_obs / bc_dim only: the cross-entropy form."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        super().__init__(obs, target, bc_obs, bc_dim, loss="cross_entropy")


def regression_data():
    g = torch.Generator().manual_seed(81)
    return torch.randn(4, 5, 3, generator=g), (torch.rand(4, 5, 2, generator=g) * 1.6 - 0.8)


def run(cell, out_tanh, cls, agent, dims, P, sigma, n_gen, table, noise_seed, obs, target, **kw):
    mg.MLP = policy_class(cell, out_tanh)
    mg.SynthAgent = agent
    # run_reference sizes each noise row with orc.mlp_param_count(dims): give it the recurrent policy's count
    orc = mg.orc
    mg.orc = types.SimpleNamespace(mlp_param_count=lambda d: param_count(cell, d), noise_offsets=orc.noise_offsets)
    try:
        return mg.run_reference(cls, list(dims), P, sigma, n_gen, table, noise_seed, obs, target, **kw)
    finally:
        mg.orc = orc


def main():
    obs, target = regression_data()
    out = run("gru", True, mg.ref.ES, SequenceAgent, (3, 16, 2), 16, 0.05, 3, mg.make_table(1 << 14, 81), 61,
              obs, target)
    np.savez_compressed(os.path.join(HERE, "es_seq_gru_p16.npz"), **out)
    obs, target = recall_dataset()
    out = run("lstm", False, mg.ref.NSR_ES, SequenceXent, (4, 8, 3), 8, 0.02, 4, mg.make_table(1 << 14, 82), 67,
              obs, target, bc_obs=3, bc_dim=54)
    np.savez_compressed(os.path.join(HERE, "nsr_seq_lstm_p8.npz"), **out)
    for f in ("es_seq_gru_p16.npz", "nsr_seq_lstm_p8.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
