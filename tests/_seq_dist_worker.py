"""Worker for tests/test_rnn_sequence_cpu.py: one rank of a world_size-N gloo job running the fused ES host logic
for a recurrent policy on a SequenceAgent, with the oracle stand-in backend.  Writes its final state."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import estorch_b200 as E  # noqa: E402
from _rnn_oracle import policy_class  # noqa: E402
from _seq_oracle import SeqOracleBackend  # noqa: E402


def run():
    g = torch.Generator().manual_seed(9)
    obs, tgt = torch.randn(5, 4, 3, generator=g), torch.rand(5, 4, 2, generator=g) - 0.5
    torch.manual_seed(31)
    be = SeqOracleBackend()
    es = E.ES(policy_class("gru", True), E.SequenceAgent, torch.optim.Adam, population_size=16, sigma=0.05,
              policy_kwargs={"dims": (3, 8, 2)}, agent_kwargs=dict(obs=obs, target=tgt),
              optimizer_kwargs={"lr": 0.02}, noise_table_size=1 << 13, noise_seed=5, _backend=be)
    es.log = lambda: None
    assert es._fused and es._is_rnn and not es._population
    es.train(n_steps=3)
    return es, be


def main():
    es, be = run()
    np.savez(os.path.join(sys.argv[1], f"rank{es.rank}.npz"), theta=es._slots[0].theta.numpy(),
             returns=es.population_returns, world=es.n_workers, pairs_local=es._pairs_local,
             episode=float(es.episode_reward), seq_calls=be.seq_calls)


if __name__ == "__main__":
    main()
