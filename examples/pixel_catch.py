"""Catch from pixels, trained by ES in population mode with the reference's Atari policy.

The game is bsuite's Catch: a ball falls one row per step down a 10 x 5 grid, and a paddle on the bottom row
moves left, stays or moves right (3 actions); the episode ends when the ball reaches the bottom row, with
reward +1 for a catch and -1 for a miss.  Every environment is a tensor row on the GPU: the grid is rendered
into 84 x 84 frames and stacked 4 deep, so the policy sees what the reference's Atari example feeds its
network (examples/atari.py:40-76), and it acts by the argmax of its logits (examples/atari.py:62).

The policy is the reference's Atari ``Policy`` (conv + VirtualBatchNorm, examples/atari.py:14-37), with its
reference batch collected from random-action episodes as the reference collects its own
(examples/atari.py:89-120).  ``ES`` selects population mode for a ``PopulationAgent`` on one GPU: every
environment step of all P members (each playing ``EPISODES`` games side by side) is one CUDA launch, and the
members' VBN statistics are one more launch per generation.

    python examples/pixel_catch.py [--generations 30] [--population 256]
"""
import argparse
import random

import torch
from torch import nn
from torch.nn import functional as F

from estorch_b200 import ES, PopulationAgent, VirtualBatchNorm

ROWS, COLS, STACK, CELL_H, CELL_W = 10, 5, 4, 8, 16
EPISODES = 4                # games per member and generation, played side by side (the B of act)
# tests/test_population_conv_gpu.py: on one H100 (seed 0) the mean reward went from -0.60 (generation 0) to 0.40
# (mean of the last three of 30 generations); the test asks for a gain of at least TEST_MARGIN
TEST_GENERATIONS, TEST_POPULATION, TEST_MARGIN = 30, 256, 0.5


class Policy(nn.Module):
    """examples/atari.py:14-37, with this package's VirtualBatchNorm."""

    def __init__(self, n_actions, xref):
        super().__init__()
        self.xref = xref
        self.conv1 = nn.Conv2d(4, 16, 8, 4)
        self.bn1 = VirtualBatchNorm(16)
        self.conv2 = nn.Conv2d(16, 32, 4, 2)
        self.bn2 = VirtualBatchNorm(32)
        self.fc1 = nn.Linear(2592, 256)
        self.fc2 = nn.Linear(256, n_actions)

    def forward(self, x):
        xref = F.relu(self.bn1(self.conv1(self.xref)))
        F.relu(self.bn2(self.conv2(xref)))
        x = F.relu(self.bn1(self.conv1(x)))
        x = F.relu(self.bn2(self.conv2(x)))
        x = F.relu(self.fc1(x.view(-1, 2592)))
        return self.fc2(x)


def render(ball_r, ball_c, paddle):
    """[N] ball row / column and paddle column -> [N, 84, 84] frames (ball 1.0, paddle 0.5)."""
    N, dev = ball_r.shape[0], ball_r.device
    img = torch.zeros(N, 84, 84, device=dev)
    ys = torch.arange(84, device=dev)[None, :, None]
    xs = torch.arange(84, device=dev)[None, None, :]
    y0, x0 = 2, 2

    def cell(r, c):
        top, left = y0 + r[:, None, None] * CELL_H, x0 + c[:, None, None] * CELL_W
        return (ys >= top) & (ys < top + CELL_H) & (xs >= left) & (xs < left + CELL_W)
    img = torch.where(cell(torch.full_like(paddle, ROWS - 1), paddle), torch.full_like(img, 0.5), img)
    return torch.where(cell(ball_r, ball_c), torch.ones_like(img), img)


def play(policy_fn, members, episodes, generator, device, random_actions=False, frames_out=None):
    """``members`` x ``episodes`` games side by side; ``policy_fn`` maps [members, episodes, 4, 84, 84] frames to
    [members, episodes, 3] logits.  Returns the mean reward per member."""
    N = members * episodes
    ball_c = torch.randint(0, COLS, (N,), generator=generator, device=device)
    ball_r = torch.zeros(N, dtype=torch.long, device=device)
    paddle = torch.full((N,), COLS // 2, dtype=torch.long, device=device)
    stack = render(ball_r, ball_c, paddle)[:, None].repeat(1, STACK, 1, 1)
    for _ in range(ROWS - 1):
        if frames_out is not None:
            frames_out.append(stack.clone())
        if random_actions:
            a = torch.randint(0, 3, (N,), generator=generator, device=device)
        else:
            a = policy_fn(stack.view(members, episodes, STACK, 84, 84)).reshape(N, 3).argmax(1)
        paddle = (paddle + a - 1).clamp(0, COLS - 1)
        ball_r = ball_r + 1
        stack = torch.cat([stack[:, 1:], render(ball_r, ball_c, paddle)[:, None]], 1)
    reward = torch.where(paddle == ball_c, 1.0, -1.0)
    return reward.view(members, episodes).mean(1)


def reference_batch(n=128, seed=0, device="cpu"):
    """n frames sampled from random-action games (examples/atari.py:89-120)."""
    g = torch.Generator(device=device).manual_seed(seed)
    frames = []
    play(None, 64, 1, g, device, random_actions=True, frames_out=frames)
    frames = torch.cat(frames)
    pick = random.Random(seed).sample(range(frames.shape[0]), n)
    return frames[pick].contiguous().cpu()


class Catch(PopulationAgent):
    """Catch games of all members at once; the ball columns come from a generator seeded once."""

    def __init__(self, seed=0):
        self.seed = seed
        self._gen = None

    def rollout_population(self, act, members):
        if self._gen is None or self._gen.device != torch.device(self.device):
            self._gen = torch.Generator(device=self.device).manual_seed(self.seed)
        return play(act, members, EPISODES, self._gen, self.device)

    def rollout(self, policy):
        """The reference protocol (hooks mode): the plain policy takes [N, 4, 84, 84] frames."""
        dev = next(policy.parameters()).device
        if self._gen is None or self._gen.device != dev:
            self._gen = torch.Generator(device=dev).manual_seed(self.seed)
        with torch.no_grad():
            ret = play(lambda o: policy(o.reshape(-1, STACK, 84, 84)).view(1, EPISODES, 3), 1, EPISODES, self._gen, dev)
        return float(ret[0])


def train(generations=30, population_size=256, seed=0, backend=None, verbose=True):
    """Train with ES in population mode; returns the mean population reward of every generation."""
    torch.manual_seed(seed)
    xref = reference_batch(seed=seed)
    means = []
    es = ES(Policy, Catch, torch.optim.Adam, population_size=population_size, sigma=0.02,
            policy_kwargs={"n_actions": 3, "xref": xref}, agent_kwargs={"seed": seed},
            optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 24, noise_seed=seed + 1, _backend=backend)
    if not es._population:
        raise RuntimeError("population mode needs one CUDA GPU and the conv + VBN policy")

    def log():
        means.append(float(es.population_returns.mean()))
        if verbose:
            print(f"generation {es.step:3d}  mean reward {means[-1]:+.3f}  theta's reward {es.episode_reward:+.3f}")
    es.log = log
    es.train(n_steps=generations)
    return means


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--generations", type=int, default=TEST_GENERATIONS)
    ap.add_argument("--population", type=int, default=TEST_POPULATION)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    train(a.generations, a.population, a.seed)
