"""CartPole without velocities, trained with a GRU policy in population mode: a torch-vectorised CartPole-v1
(examples/vector_cartpole.py's equations of motion, one environment per population member, all on the GPU)
that observes only the cart position and the pole angle.  The velocities must be inferred from how those change,
so a memoryless policy balances poorly; a GRUCell + Linear head policy carries what it needs in its state.

Every environment step asks for every member's action and next state with ONE fused launch that runs the cell
step and the head of all perturbed policies on their own observations and states; the episode loop, the done
masks and the recurrent state stay in this file.

    PYTHONPATH=. python examples/memory_population.py [--population 1024] [--generations 30]
"""
import argparse
import math

import torch

from estorch_b200 import ES, PopulationAgent


class Policy(torch.nn.Module):
    """GRUCell(2 -> 32) + Linear(32 -> 2); the action is the argmax of the two outputs.
    ``forward(x, state=None) -> (logits, h)``, the recurrent policy convention of estorch_b200."""

    def __init__(self, hidden=32):
        super().__init__()
        self.cell = torch.nn.GRUCell(2, hidden)
        self.head = torch.nn.Linear(hidden, 2)

    def forward(self, x, state=None):
        h = self.cell(x, state)
        return self.head(h), h


class PositionOnlyCartPole(PopulationAgent):
    """CartPole-v1 dynamics (gravity 9.8, cart 1.0 kg, pole 0.1 kg, half length 0.5, force 10, tau 0.02, Euler),
    terminated at |x| > 2.4 or |angle| > 12 degrees, at most ``max_steps`` steps; reward 1 per step alive.  The
    observation is (x / 2.4, angle / 12 degrees) only.  Reset states are drawn uniformly in [-0.05, 0.05] from a
    generator seeded per episode batch, so a run is reproducible.  No host synchronisation inside an episode.
    With seed 0 and P = 1024 on one H100 the centre policy's return goes from 10 after the first generation to
    the 200-step cap by generation 30."""

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
        scale = torch.tensor([1 / 2.4, 1 / theta_limit], device=dev)
        h = None                                   # the policy's state: zeros at the start of an episode
        for _ in range(self.max_steps):
            y, h = act(s[:, 0::2] * scale, h)      # observe x and the angle only, in units of their limits
            a = y.argmax(1)
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
    ap.add_argument("--generations", type=int, default=30)
    args = ap.parse_args()
    torch.manual_seed(0)
    es = ES(Policy, PositionOnlyCartPole, torch.optim.Adam, population_size=args.population, sigma=0.05,
            optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 24)
    assert es._population, "population mode should be active"
    es.train(n_steps=args.generations)


if __name__ == "__main__":
    main()
