"""Drop-in check: the reference's own example scripts run against this package.

The scripts are READ at test time from oracle/_ref/examples, where ``__graft_entry__.build()``
installs the reference (never copied into the repo's sources; the tests skip where build() had no
reference source tree to install).  They are
executed with ``import estorch`` resolving to ``estorch_b200``, a stand-in ``gym`` (the image
has no gym) and the CPU stand-in backend of tests/_oracle_backend.py.  Only the launch
parameters are rewritten (``n_proc=2`` would re-exec under torchrun, hundreds of steps
are cut to a few) -- the classes, hooks and attribute accesses are the reference's text.
"""
import math
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

import estorch_b200
from _oracle_backend import OracleBackend
from oracle.ref_shim import REF_EXAMPLES as EXAMPLES

pytestmark = pytest.mark.skipif(not os.path.isdir(EXAMPLES), reason="build() installed no reference examples here")


class _Space:
    def __init__(self, shape=None, n=None):
        self.shape, self.n = shape, n


class CartPoleStandIn:
    """Textbook cart-pole (Barto, Sutton & Anderson 1983 equations, Euler steps of 20 ms) with
    the pre-0.26 gym protocol the reference examples use: reset() -> obs,
    step(a) -> (obs, reward, done, info); episodes end at |x| > 2.4, |angle| > 12 deg or 500 steps."""
    gravity, m_cart, m_pole, half_len, force, tau = 9.8, 1.0, 0.1, 0.5, 10.0, 0.02

    def __init__(self, seed=0):
        self.observation_space, self.action_space = _Space(shape=(4,)), _Space(n=2)
        self.rng = np.random.RandomState(seed)
        self.state, self.t = None, 0

    def reset(self):
        self.state, self.t = self.rng.uniform(-0.05, 0.05, size=4), 0
        return self.state.astype(np.float32)

    def step(self, action):
        x, x_dot, th, th_dot = self.state
        f = self.force if int(action) == 1 else -self.force
        total_m, pm_l = self.m_cart + self.m_pole, self.m_pole * self.half_len
        tmp = (f + pm_l * th_dot ** 2 * math.sin(th)) / total_m
        th_acc = (self.gravity * math.sin(th) - math.cos(th) * tmp) / \
                 (self.half_len * (4.0 / 3.0 - self.m_pole * math.cos(th) ** 2 / total_m))
        x_acc = tmp - pm_l * th_acc * math.cos(th) / total_m
        self.state = np.array([x + self.tau * x_dot, x_dot + self.tau * x_acc,
                               th + self.tau * th_dot, th_dot + self.tau * th_acc])
        self.t += 1
        done = bool(abs(self.state[0]) > 2.4 or abs(self.state[2]) > 12 * math.pi / 180 or self.t >= 500)
        return self.state.astype(np.float32), 1.0, done, {}

    def render(self):
        pass


class WalkerStandIn:
    """A 24-observation / 4-action continuous-control stand-in with the shape of BipedalWalker-v3
    (examples/nsra_es.py): a damped linear system pushed by the actions; 40-70 steps per episode,
    reward = forward velocity minus an action cost."""

    def __init__(self, seed=0):
        self.observation_space, self.action_space = _Space(shape=(24,)), _Space(shape=(4,))
        self.rng = np.random.RandomState(seed)
        self.mix = self.rng.standard_normal((4, 24)).astype(np.float32) * 0.3

    def reset(self):
        self.state = self.rng.uniform(-0.1, 0.1, size=24).astype(np.float32)
        self.t, self.horizon = 0, int(self.rng.randint(40, 71))
        return self.state.copy()

    def step(self, action):
        a = np.clip(np.asarray(action, dtype=np.float32).reshape(4), -1.0, 1.0)
        self.state = (0.9 * self.state + a @ self.mix).astype(np.float32)
        self.t += 1
        return self.state.copy(), float(self.state[0] - 0.01 * np.sum(a * a)), self.t >= self.horizon, {}

    def render(self):
        pass


@pytest.fixture
def reference_world(monkeypatch):
    """``import estorch`` -> this package (CPU stand-in backend), ``import gym`` -> the stand-in,
    the examples directory importable (early_stopping.py / custom_es.py import cartpole_es)."""
    gym = types.ModuleType("gym")
    gym.make = lambda name: CartPoleStandIn() if name.startswith("CartPole") else WalkerStandIn()
    monkeypatch.setitem(sys.modules, "gym", gym)
    monkeypatch.setitem(sys.modules, "estorch", estorch_b200)
    monkeypatch.syspath_prepend(EXAMPLES)
    sys.modules.pop("cartpole_es", None)
    real_init = estorch_b200.ES.__init__

    def init_with_cpu_backend(self, *a, **kw):
        kw.setdefault("_backend", OracleBackend())
        kw.setdefault("noise_table_size", 1 << 16)
        real_init(self, *a, **kw)
    monkeypatch.setattr(estorch_b200.ES, "__init__", init_with_cpu_backend)
    yield
    sys.modules.pop("cartpole_es", None)


def _run_example(name, n_steps, population=8):
    src = open(os.path.join(EXAMPLES, name)).read()
    src, n1 = re.subn(r"n_proc=\d+", "n_proc=1", src)
    src, n2 = re.subn(r"n_steps=\d+", f"n_steps={n_steps}", src)
    src, n3 = re.subn(r"population_size=\d+", f"population_size={population}", src)
    assert n1 == 1 and n2 == 1 and n3 == 1, "the example's launch line changed upstream"
    scope = {"__name__": "__main__", "__file__": os.path.join(EXAMPLES, name)}
    exec(compile(src, os.path.join(EXAMPLES, name), "exec"), scope)
    return scope


def test_cartpole_example_runs_unmodified(reference_world, capsys):
    """examples/cartpole_es.py: ES(Policy, Agent, Adam, ...).train(), then es.policy and
    es.best_policy_dict feed the user's own rollout (estorch.py:108-117 attributes)."""
    scope = _run_example("cartpole_es.py", n_steps=2)
    es = scope["es"]
    assert type(es).__name__ == "ES" and not es._fused        # a gym-style host agent: hooks path
    assert es.step == 2 and es.population_returns.shape == (8, 1) and es.population_returns.dtype == np.float32
    assert set(es.best_policy_dict) == set(scope["Policy"](4, 2).state_dict())
    out = capsys.readouterr().out
    assert "Latest Policy Reward" in out and "Best Policy Reward" in out and "Episode Reward" in out


def test_early_stopping_example_runs_unmodified(reference_world, capsys):
    """examples/early_stopping.py overrides log(), indexes population_parameters by member and
    calls terminate() (estorch.py:150-152): make every episode 'perfect' so that it triggers."""
    import cartpole_es                                            # the reference's module, via syspath
    monkey_reward = 500.0
    cartpole_es.Agent.rollout = lambda self, policy, render=False: monkey_reward
    scope = _run_example("early_stopping.py", n_steps=5)
    es = scope["es"]
    assert es.step == 1                                            # stopped after the first generation
    assert tuple(es.best.shape) == (es.n_parameters,)
    assert "Reward: 500" in capsys.readouterr().out


def test_custom_es_example_runs_unmodified(reference_world, capsys):
    """examples/custom_es.py overrides _sample_policy / _calculate_grad and imports
    rank_transformation from the package: the engine must honour the overrides."""
    scope = _run_example("custom_es.py", n_steps=2)
    es = scope["es"]
    assert type(es).__name__ == "SymmetricES" and not es._fused
    assert es.step == 2 and torch.isfinite(torch.nn.utils.parameters_to_vector(es.policy.parameters())).all()
    assert "Best Policy Reward" in capsys.readouterr().out


def test_nsra_example_runs_unmodified(reference_world, capsys):
    """examples/nsra_es.py: rollout -> (reward, behaviour characterisation), the archive /
    meta-population / adaptive weight of estorch.py:388-472,623-662, es.meta_population and
    es.best_policy_dict afterwards."""
    np.random.seed(0)
    scope = _run_example("nsra_es.py", n_steps=2, population=8)
    es = scope["es"]
    assert type(es).__name__ == "NSRA_ES" and len(es.meta_population) == 3
    assert es.population_returns.shape == (8, 2) and len(es._archive) == 3 + 2    # +1 behaviour per generation
    assert not hasattr(es, "policy")                                              # as in the reference (estorch.py:135-137)
    assert 0.0 <= es.weight <= 1.0
    out = capsys.readouterr().out
    assert "Reward of 2. policy from the meta population" in out and "Best Policy Reward" in out
