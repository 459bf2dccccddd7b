"""Worker for tests/test_minibatch_cpu.py: one rank of a world_size-N gloo job running the fused ES host logic
with a sampling DeviceAgent on the oracle stand-in backend.  Writes its final state."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import estorch_b200 as E  # noqa: E402
from _batch_oracle import dataset  # noqa: E402
from _mlp_oracle import MLP  # noqa: E402
from _oracle_backend import OracleBackend  # noqa: E402


def run():
    x, y = dataset(45, 4, 3, seed=12)
    torch.manual_seed(31)
    be = OracleBackend()
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=16, sigma=0.05,
              policy_kwargs={"dims": [4, 8, 3]}, agent_kwargs=dict(obs=x, target=y, batch_size=10, batch_seed=6),
              optimizer_kwargs={"lr": 0.02}, noise_table_size=1 << 13, noise_seed=5, _backend=be)
    es.log = lambda: None
    assert es._fused and es._sampling
    es.train(n_steps=3)
    return es, be


def main():
    es, be = run()
    np.savez(os.path.join(sys.argv[1], f"rank{es.rank}.npz"), theta=es._slots[0].theta.numpy(),
             returns=es.population_returns, world=es.n_workers, episode=float(es.episode_reward),
             batch_calls=be.batch_calls)


if __name__ == "__main__":
    main()
