"""Evaluate time and training rate of ELU / SiLU / LeakyReLU MLP policies next to ReLU and Tanh
(one JSON line per measurement).

    python tools/act_ext_bench.py eval  [--acts relu,tanh,elu,silu,leaky_relu] [--modes f16,bf16,bf16s,fp32]
                                        [--iters N] [--repeats R]
    python tools/act_ext_bench.py train [--hidden silu] [--shape cartpole|north_star] [--steps K] [--warmup W]
                                        [--hooks-steps H]

``eval`` times the MLP evaluate launch alone at the north star (P = 4096, n = 1,001,760, B = 256; CUDA
events, ms per launch) for each hidden activation and precision mode, all in one session and
interleaved per repeat, so the kinds are compared under the same clocks.  ``train`` times ``ES.train``
generations of a policy with the given hidden activation through the public API twice: fused (the
engine recognises the policy) and in hooks mode (the same rollout behind a host agent, one host
rollout per member).  The card name and power limit are printed with the numbers.
"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from act_bench import MLP_1M, SHAPES, card, emit  # noqa: E402

HIDDEN_CODES = {"relu": 0, "tanh": 1, "elu": 3, "silu": 4, "leaky_relu": 5}   # include/estk.h ESTK_ACT_*
MODULES = {"relu": torch.nn.ReLU, "tanh": torch.nn.Tanh, "elu": torch.nn.ELU, "silu": torch.nn.SiLU,
           "leaky_relu": torch.nn.LeakyReLU}


def eval_times(args):
    from estorch_b200.backend import CudaBackend
    be = CudaBackend(torch.device("cuda", 0))
    dims, pairs, B = MLP_1M, 2048, 256
    n = sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))
    table = be.alloc(1 << 28)
    be.fill_noise_table(table, 42)
    offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
    torch.manual_seed(0)
    theta = torch.randn(n, device=be.device) * 0.05
    obs, tgt = torch.randn(B, 128, device=be.device), torch.randn(B, 288, device=be.device)
    th16, tbb = be.alloc(n, dtype=torch.bfloat16), be.alloc(table.numel(), dtype=torch.bfloat16)
    tb16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, tb16) == 0
    be.shadow_bf16(table, tbb)
    be.shadow_bf16(theta, th16)
    ret = be.zeros(2 * pairs)
    gpu = card()
    for rep in range(args.repeats):
        for a in args.acts.split(","):
            for mode in args.modes.split(","):
                kw = {"table16": tb16} if mode == "f16" else {"theta16": th16, "table16": tbb} if mode == "bf16s" else {}
                if HIDDEN_CODES[a]:
                    kw["act"] = HIDDEN_CODES[a]

                def run():
                    be.eval_mlp(dims, theta, table, offs, order, pairs, 0.02, obs, tgt, ret[:pairs], ret[pairs:],
                                precision=mode, **kw)
                for _ in range(3):
                    run()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    run()
                e1.record()
                torch.cuda.synchronize()
                emit(what="eval", act=a, mode=mode, ms=round(e0.elapsed_time(e1) / args.iters, 4), repeat=rep,
                     checksum=float(ret.double().sum()), gpu=gpu)


class Policy(torch.nn.Module):
    def __init__(self, dims, hidden="silu"):
        super().__init__()
        layers = []
        for i in range(len(dims) - 1):
            layers.append(torch.nn.Linear(dims[i], dims[i + 1]))
            if i + 2 < len(dims):
                layers.append(MODULES[hidden]())
        self.net = torch.nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


class HostAgent:
    """The DeviceAgent's rollout behind a plain host agent: the engine runs it in hooks mode."""
    def __init__(self, obs, target):
        import estorch_b200 as E
        self.inner = E.DeviceAgent(obs, target)

    def rollout(self, policy):
        return self.inner.rollout(policy)


def train_rate(args):
    import estorch_b200 as E
    dims = SHAPES[args.shape]
    g = torch.Generator().manual_seed(1234)
    obs, tgt = torch.randn(256, dims[0], generator=g), torch.rand(256, dims[-1], generator=g) * 1.8 - 0.9
    for agent, steps in ((E.DeviceAgent, args.steps), (HostAgent, args.hooks_steps)):
        if not steps:
            continue
        torch.manual_seed(0)
        es = E.ES(Policy, agent, torch.optim.Adam, population_size=args.population, sigma=0.02,
                  policy_kwargs={"dims": dims, "hidden": args.hidden}, agent_kwargs=dict(obs=obs, target=tgt),
                  optimizer_kwargs={"lr": 0.01}, log_interval=10 ** 9)
        es.log = lambda: None
        if args.warmup:
            es.train(n_steps=args.warmup if es._fused else 1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        es.train(n_steps=steps)
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        emit(what="train", shape=args.shape, hidden=args.hidden, population=args.population, fused=bool(es._fused),
             precision=es._precision, steps=steps, seconds=round(s, 4), generations_per_s=round(steps / s, 4),
             episode_reward=float(es.episode_reward), gpu=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["eval", "train"])
    ap.add_argument("--acts", default="relu,tanh,elu,silu,leaky_relu")
    ap.add_argument("--modes", default="f16,bf16,bf16s,fp32")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--shape", default="cartpole", choices=sorted(SHAPES))
    ap.add_argument("--hidden", default="silu", choices=sorted(HIDDEN_CODES))
    ap.add_argument("--population", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--hooks-steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    eval_times(args) if args.what == "eval" else train_rate(args)


if __name__ == "__main__":
    main()
