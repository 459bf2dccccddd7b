"""Train a small CNN image classifier with ES on the device, in fused mode.

The task is generated in code (no download): 1x28x28 images of noise with a bright bar that is horizontal,
vertical, or on one of the two diagonals; the class is the bar's orientation.  The policy is an ordinary
``nn.Sequential`` of Conv2d / ReLU / Flatten / Linear, and ``DeviceAgent(loss="cross_entropy")`` scores it on a
fixed batch.  The engine recognises the Conv2d stack and evaluates every perturbed member in one fp32 kernel
launch per generation (estk_eval_cnn.cu); no member is materialised.

    python examples/cnn_classifier.py [--generations 30] [--population 512]
"""
import argparse
import os
import sys

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from estorch_b200 import ES, DeviceAgent  # noqa: E402

# the test runs these settings and asks for a gain in training accuracy of at least TEST_MARGIN
TEST_GENERATIONS, TEST_POPULATION, TEST_MARGIN = 30, 512, 0.3


def bars(n, seed, size=28):
    """[n, 1, size, size] images and [n, 4] one-hot targets: a bar of one of four orientations on noise."""
    g = torch.Generator().manual_seed(seed)
    x = 0.2 * torch.rand(n, 1, size, size, generator=g)
    labels = torch.randint(0, 4, (n,), generator=g)
    centre = torch.randint(8, size - 8, (n, 2), generator=g)
    t = torch.arange(-6, 7)
    for i in range(n):
        r, c = int(centre[i, 0]), int(centre[i, 1])
        dr, dc = [(0, 1), (1, 0), (1, 1), (1, -1)][int(labels[i])]
        x[i, 0, r + dr * t, c + dc * t] = 1.0
    return x, nn.functional.one_hot(labels, 4).float()


class Classifier(nn.Module):
    def __init__(self):
        super().__init__()
        self.net = nn.Sequential(nn.Conv2d(1, 8, 5, stride=2, padding=2), nn.ReLU(),
                                 nn.Conv2d(8, 16, 5, stride=2, padding=2), nn.ReLU(),
                                 nn.Flatten(), nn.Linear(16 * 7 * 7, 4))

    def forward(self, x):
        return self.net(x)


def accuracy(policy, x, y):
    with torch.no_grad():
        p = next(policy.parameters())
        return float((policy(x.to(p.device)).argmax(1).cpu() == y.argmax(1)).float().mean())


def main(generations=TEST_GENERATIONS, population=TEST_POPULATION, seed=0, verbose=False, eval_precision="auto"):
    """Returns (first centre return, last centre return, accuracy before, accuracy after) on the batch.
    ``eval_precision="tf32"`` evaluates on TF32 tensor cores instead of fp32."""
    torch.manual_seed(seed)
    x, y = bars(256, seed)
    es = ES(Classifier, DeviceAgent, torch.optim.Adam, population_size=population, sigma=0.02,
            agent_kwargs=dict(obs=x, target=y, loss="cross_entropy"), optimizer_kwargs={"lr": 0.01},
            eval_precision=eval_precision)
    assert es._fused, "the CNN should be evaluated by the fused kernel"
    acc0 = accuracy(es.policy, x, y)
    rewards = []

    def log():
        rewards.append(float(es.episode_reward))
        if verbose:
            print(f"generation {es.step}: centre return {rewards[-1]:.4f}")
    es.log = log
    es.train(n_steps=generations)
    return rewards[0], rewards[-1], acc0, accuracy(es.policy, x, y)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--generations", type=int, default=TEST_GENERATIONS)
    ap.add_argument("--population", type=int, default=TEST_POPULATION)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--eval-precision", default="auto", choices=["auto", "fp32", "tf32"])
    a = ap.parse_args()
    first, last, acc0, acc1 = main(a.generations, a.population, a.seed, verbose=True, eval_precision=a.eval_precision)
    print(f"centre return {first:.4f} -> {last:.4f}, accuracy {acc0:.3f} -> {acc1:.3f}")
