"""CartPole trained in population mode: a torch-vectorised CartPole-v1 (the classic-control equations of
motion, one environment per population member, all on the GPU) behind estorch_b200.PopulationAgent.

Every environment step asks for every member's action with ONE fused launch that evaluates all perturbed
policies on their own observations; the episode loop, done masks and returns stay in this file.

    python examples/vector_cartpole.py [--population 1024] [--generations 20]
"""
import argparse
import math

import torch

from estorch_b200 import ES, PopulationAgent


class Policy(torch.nn.Module):
    """4-64-64-2 ReLU MLP; the action is the argmax of the two outputs (examples/cartpole_es.py)."""

    def __init__(self):
        super().__init__()
        self.linear_1 = torch.nn.Linear(4, 64)
        self.activation_1 = torch.nn.ReLU()
        self.linear_2 = torch.nn.Linear(64, 64)
        self.activation_2 = torch.nn.ReLU()
        self.linear_3 = torch.nn.Linear(64, 2)

    def forward(self, x):
        return self.linear_3(self.activation_2(self.linear_2(self.activation_1(self.linear_1(x)))))


class VectorCartPole(PopulationAgent):
    """CartPole-v1 dynamics (gravity 9.8, cart 1.0 kg, pole 0.1 kg, half length 0.5, force 10, tau 0.02, Euler),
    terminated at |x| > 2.4 or |angle| > 12 degrees, at most ``max_steps`` steps; reward 1 per step alive.
    Reset states are drawn uniformly in [-0.05, 0.05] from a generator seeded per episode batch, so a run is
    reproducible.  No host synchronisation inside an episode: the done mask is a tensor."""

    def __init__(self, max_steps=200, seed=0):
        self.max_steps = max_steps
        self.seed = seed
        self.episodes = 0

    def rollout_population(self, act, members):
        dev = self.device
        g = torch.Generator(device=dev).manual_seed(self.seed * 1000003 + self.episodes)
        self.episodes += 1
        s = (torch.rand(members, 4, generator=g, device=dev) - 0.5) * 0.1
        alive = torch.ones(members, device=dev)
        ret = torch.zeros(members, device=dev)
        gravity, mc, mp, length, force_mag, tau = 9.8, 1.0, 0.1, 0.5, 10.0, 0.02
        total, pml = mc + mp, mp * length
        theta_limit = 12 * 2 * math.pi / 360
        for _ in range(self.max_steps):
            a = act(s).argmax(1)
            x, x_dot, th, th_dot = s.unbind(1)
            force = (a.float() * 2 - 1) * force_mag
            cos, sin = torch.cos(th), torch.sin(th)
            temp = (force + pml * th_dot * th_dot * sin) / total
            th_acc = (gravity * sin - cos * temp) / (length * (4.0 / 3.0 - mp * cos * cos / total))
            x_acc = temp - pml * th_acc * cos / total
            s = torch.stack([x + tau * x_dot, x_dot + tau * x_acc, th + tau * th_dot, th_dot + tau * th_acc], 1)
            ret = ret + alive
            alive = alive * ((s[:, 0].abs() <= 2.4) & (s[:, 2].abs() <= theta_limit)).float()
        return ret


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--population", type=int, default=1024)
    ap.add_argument("--generations", type=int, default=20)
    args = ap.parse_args()
    torch.manual_seed(0)
    es = ES(Policy, VectorCartPole, torch.optim.Adam, population_size=args.population, sigma=0.02,
            optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 24)
    assert es._population, "population mode should be active"
    es.train(n_steps=args.generations)


if __name__ == "__main__":
    main()
