"""Delayed recall, trained with a GRU policy on a fixed batch of sequences: each sequence shows one of K cues at its
first step, blank observations for ``delay`` steps, then a recall flag, and the policy must name the cue at the
last step.  Only that step is scored (the cross-entropy target rows of the other steps are all zeros), so a
policy without memory cannot do better than guessing: -log(K) / T.

``SequenceAgent`` declares the batch; with Adam, ``ES`` runs the fused generation, in which ONE launch evaluates
every perturbed policy over all B sequences and T steps, with each member's state kept on chip across the steps.

    PYTHONPATH=. python examples/sequence_recall.py [--population 256] [--generations 60] [--delay 8]
"""
import argparse
import math

import torch

from estorch_b200 import ES, SequenceAgent


class Policy(torch.nn.Module):
    """GRUCell(K + 1 -> 32) + Linear(32 -> K): the logits of the cue.
    ``forward(x, state=None) -> (logits, h)``, the recurrent policy convention of estorch_b200."""

    def __init__(self, cues=4, hidden=32):
        super().__init__()
        self.cell = torch.nn.GRUCell(cues + 1, hidden)
        self.head = torch.nn.Linear(hidden, cues)

    def forward(self, x, state=None):
        h = self.cell(x, state)
        return self.head(h), h


def recall_batch(cues, delay, copies):
    """obs [B, T, cues + 1] and the cross-entropy target [B, T, cues], B = cues * copies, T = delay + 2."""
    T, B = delay + 2, cues * copies
    obs, target = torch.zeros(B, T, cues + 1), torch.zeros(B, T, cues)
    for b in range(B):
        obs[b, 0, b % cues] = 1.0
        obs[b, T - 1, cues] = 1.0
        target[b, T - 1, b % cues] = 1.0
    return obs, target


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--population", type=int, default=256)
    ap.add_argument("--generations", type=int, default=60)
    ap.add_argument("--cues", type=int, default=4)
    ap.add_argument("--delay", type=int, default=8)
    args = ap.parse_args()
    obs, target = recall_batch(args.cues, args.delay, copies=4)
    torch.manual_seed(0)
    es = ES(Policy, SequenceAgent, torch.optim.Adam, population_size=args.population, sigma=0.05,
            policy_kwargs={"cues": args.cues}, agent_kwargs=dict(obs=obs, target=target, loss="cross_entropy"),
            optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 22)
    assert es._fused and es._is_rnn, "the fused sequence evaluate should be active"
    print(f"a policy without memory scores at best {-math.log(args.cues) / (args.delay + 2):.4f}")
    es.train(n_steps=args.generations)


if __name__ == "__main__":
    main()
