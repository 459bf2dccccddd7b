"""Train an MLP classifier with ES on minibatches of a 60,000-row dataset, drawn on the device.

The dataset is generated in code (no download): 784-D points around ten class means, one-hot targets.  The
agent holds all of it, ``DeviceAgent(..., loss="cross_entropy", batch_size=256)``, and every generation scores all
perturbed members on the same fresh minibatch of 256 rows.  The engine keeps the dataset on the GPU and gathers
each generation's rows in one kernel launch at the head of the generation (estk_batch.cu), so the host plays no
part and the generation still replays from a CUDA graph.  Accuracy is reported on the whole dataset.

    python examples/minibatch_classifier.py [--rows 60000] [--generations 60] [--population 1024]
"""
import argparse
import os
import sys

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from estorch_b200 import ES, DeviceAgent  # noqa: E402

# the test runs these settings and asks for a full-dataset accuracy of at least TEST_ACCURACY afterwards
TEST_SETTINGS = dict(rows=60000, generations=60, population=1024, batch_size=256)
TEST_ACCURACY = 0.6


def class_conditional(n, seed, dim=784, classes=10, separation=0.15):
    """[n, dim] points drawn around ``classes`` random means (unit noise per coordinate) and [n, classes] one-hot
    targets."""
    g = torch.Generator().manual_seed(seed)
    means = separation * torch.randn(classes, dim, generator=g)
    labels = torch.randint(0, classes, (n,), generator=g)
    x = means[labels] + torch.randn(n, dim, generator=g)
    return x, nn.functional.one_hot(labels, classes).float()


class Classifier(nn.Module):
    def __init__(self, dim=784, hidden=64, classes=10):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(dim, hidden), nn.ReLU(), nn.Linear(hidden, classes))

    def forward(self, x):
        return self.net(x)


def accuracy(policy, x, y):
    with torch.no_grad():
        p = next(policy.parameters())
        return float((policy(x.to(p.device)).argmax(1).cpu() == y.argmax(1)).float().mean())


def main(rows=60000, generations=60, population=1024, batch_size=256, seed=0, verbose=False):
    """Returns the full-dataset accuracy before and after training."""
    torch.manual_seed(seed)
    x, y = class_conditional(rows, seed)
    es = ES(Classifier, DeviceAgent, torch.optim.Adam, population_size=population, sigma=0.02,
            agent_kwargs=dict(obs=x, target=y, loss="cross_entropy", batch_size=batch_size, batch_seed=seed),
            optimizer_kwargs={"lr": 0.01})
    assert es._fused and es._sampling, "the minibatches should be drawn by the fused generation"
    acc0 = accuracy(es.policy, x, y)

    def log():
        if verbose and (es.step + 1) % 10 == 0:
            print(f"generation {es.step + 1}: minibatch return {float(es.episode_reward):.4f}, "
                  f"full-dataset accuracy {accuracy(es.policy, x, y):.3f}")
    es.log = log
    es.train(n_steps=generations)
    return acc0, accuracy(es.policy, x, y)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=TEST_SETTINGS["rows"])
    ap.add_argument("--generations", type=int, default=TEST_SETTINGS["generations"])
    ap.add_argument("--population", type=int, default=TEST_SETTINGS["population"])
    ap.add_argument("--batch-size", type=int, default=TEST_SETTINGS["batch_size"])
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    acc0, acc1 = main(a.rows, a.generations, a.population, a.batch_size, a.seed, verbose=True)
    print(f"full-dataset accuracy {acc0:.3f} -> {acc1:.3f}")
