"""Worker for tests/test_cnn_cpu.py: one rank of a world_size-N gloo job running the fused ES host logic for a
convolutional policy on a DeviceAgent, with the oracle stand-in backend.  Writes its final state."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import estorch_b200 as E  # noqa: E402
from _cnn_oracle import CnnOracleBackend, image_task, pack, policy_class  # noqa: E402


def run():
    obs, tgt = image_task(6, (1, 12, 12), seed=2)
    torch.manual_seed(31)
    be = CnnOracleBackend()
    es = E.ES(policy_class(2, "elu", True), E.DeviceAgent, torch.optim.Adam, population_size=16, sigma=0.05,
              policy_kwargs={"dims": pack((1, 12, 12), [(4, 3, 2, 1), (6, 3, 2, 0)], [8, 4])},
              agent_kwargs=dict(obs=obs, target=tgt - 0.5), optimizer_kwargs={"lr": 0.02},
              noise_table_size=1 << 13, noise_seed=5, _backend=be)
    es.log = lambda: None
    assert es._fused and es._is_cnn and not es._population
    es.train(n_steps=3)
    return es, be


def main():
    es, be = run()
    np.savez(os.path.join(sys.argv[1], f"rank{es.rank}.npz"), theta=es._slots[0].theta.numpy(),
             returns=es.population_returns, world=es.n_workers, pairs_local=es._pairs_local,
             episode=float(es.episode_reward), cnn_calls=be.cnn_calls)


if __name__ == "__main__":
    main()
