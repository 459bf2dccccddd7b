"""Catch from the raw grid, trained by ES in population mode with a plain convolutional policy.

The game is bsuite's Catch, as in examples/pixel_catch.py: a ball falls one row per step down a 10 x 5 grid, and a
paddle on the bottom row moves left, stays or moves right (3 actions); the episode ends when the ball reaches the
bottom row, with reward +1 for a catch and -1 for a miss.  Every environment is a tensor row on the GPU.  The
observation is the grid itself as a 1 x 10 x 5 image (ball 1.0, paddle 0.5), and the policy acts by the argmax
of its outputs.

The policy is a plain ``nn.Sequential`` -- Conv2d(1, 16, 3, padding=1), ReLU, Conv2d(16, 32, 3), ReLU, Flatten,
Linear(768, 64), ReLU, Linear(64, 3) -- with no VirtualBatchNorm.  The agent declares ``obs_shape = (1, 10, 5)``,
so ``ES`` recognises the Conv2d stack and selects population mode on one GPU: every environment step of all P
members (each playing ``EPISODES`` games side by side) is one CUDA launch of every perturbed policy.  The same
agent runs in hooks mode (``mode="hooks"``) and under the reference through ``rollout``.

    python examples/cnn_catch.py [--generations 60] [--population 256] [--mode population|hooks]
"""
import argparse

import torch
from torch import nn

from estorch_b200 import ES, PopulationAgent

ROWS, COLS = 10, 5
EPISODES = 4                # games per member and generation, played side by side (the B of act)
# tests/test_population_cnn_gpu.py: on one H100 80GB HBM3 at a 700 W power limit (seed 0) the mean reward went
# from -0.600 (generation 0) to +0.523 (mean of the last three of 60 generations); the test asks for a gain of at
# least TEST_MARGIN.  Over 30 generations, sigma and lr in {0.02, 0.05, 0.1, 0.2} x {0.01, 0.03, 0.1}, most
# settings had not left the flat start (a plain CNN's outputs on a sparse grid barely depend on it at first).
TEST_GENERATIONS, TEST_POPULATION, TEST_MARGIN = 60, 256, 0.5
SIGMA, LR = 0.05, 0.03


def policy():
    return nn.Sequential(nn.Conv2d(1, 16, 3, padding=1), nn.ReLU(), nn.Conv2d(16, 32, 3), nn.ReLU(), nn.Flatten(),
                         nn.Linear(32 * 8 * 3, 64), nn.ReLU(), nn.Linear(64, 3))


def render(ball_r, ball_c, paddle):
    """[N] ball row / column and paddle column -> [N, 1, 10, 5] grids (ball 1.0, paddle 0.5)."""
    N, dev = ball_r.shape[0], ball_r.device
    img = torch.zeros(N, ROWS * COLS, device=dev)
    img.scatter_(1, ((ROWS - 1) * COLS + paddle)[:, None], 0.5)
    img.scatter_(1, (ball_r * COLS + ball_c)[:, None], 1.0)
    return img.view(N, 1, ROWS, COLS)


def play(policy_fn, members, episodes, generator, device):
    """``members`` x ``episodes`` games side by side; ``policy_fn`` maps [members, episodes, 1, 10, 5] grids to
    [members, episodes, 3] outputs.  Returns the mean reward per member."""
    N = members * episodes
    ball_c = torch.randint(0, COLS, (N,), generator=generator, device=device)
    ball_r = torch.zeros(N, dtype=torch.long, device=device)
    paddle = torch.full((N,), COLS // 2, dtype=torch.long, device=device)
    for _ in range(ROWS - 1):
        obs = render(ball_r, ball_c, paddle).view(members, episodes, 1, ROWS, COLS)
        a = policy_fn(obs).reshape(N, 3).argmax(1)
        paddle = (paddle + a - 1).clamp(0, COLS - 1)
        ball_r = ball_r + 1
    reward = torch.where(paddle == ball_c, 1.0, -1.0)
    return reward.view(members, episodes).mean(1)


class Catch(PopulationAgent):
    """Catch games of all members at once; the ball columns come from a generator seeded once."""

    obs_shape = (1, ROWS, COLS)

    def __init__(self, seed=0):
        self.seed = seed
        self._gen = None

    def _generator(self, dev):
        if self._gen is None or self._gen.device != torch.device(dev):
            self._gen = torch.Generator(device=dev).manual_seed(self.seed)
        return self._gen

    def rollout_population(self, act, members):
        return play(act, members, EPISODES, self._generator(self.device), self.device)

    def rollout(self, policy):
        """The reference protocol (hooks mode): a plain Conv2d takes [N, 1, 10, 5], so the games fold into N."""
        dev = next(policy.parameters()).device
        with torch.no_grad():
            ret = play(lambda o: policy(o.reshape(-1, 1, ROWS, COLS)).view(1, EPISODES, 3), 1, EPISODES,
                       self._generator(dev), dev)
        return float(ret[0])


class HooksES(ES):
    """ES with an overridden hook, which keeps it in hooks mode: one torch module per member (for comparison)."""

    def _after_optimize(self, policy):
        super()._after_optimize(policy)


def train(generations=60, population_size=256, seed=0, backend=None, verbose=True, mode="population"):
    """Train with ES; returns (the mean population reward of every generation, the ES instance)."""
    torch.manual_seed(seed)
    means = []
    es = (ES if mode == "population" else HooksES)(
        policy, Catch, torch.optim.Adam, population_size=population_size, sigma=SIGMA, agent_kwargs={"seed": seed},
        optimizer_kwargs={"lr": LR}, noise_table_size=1 << 22, noise_seed=seed + 1, _backend=backend)
    if mode == "population" and not es._population:
        raise RuntimeError("population mode needs one CUDA GPU and a recognised policy")

    def log():
        means.append(float(es.population_returns.mean()))
        if verbose:
            print(f"generation {es.step:3d}  mean reward {means[-1]:+.3f}  theta's reward {es.episode_reward:+.3f}")
    es.log = log
    es.train(n_steps=generations)
    return means, es


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--generations", type=int, default=TEST_GENERATIONS)
    ap.add_argument("--population", type=int, default=TEST_POPULATION)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--mode", choices=("population", "hooks"), default="population")
    a = ap.parse_args()
    train(a.generations, a.population, a.seed, mode=a.mode)
