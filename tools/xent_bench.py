"""Cost of the cross-entropy objective (one JSON line per measurement).

    python tools/xent_bench.py eval  [--modes f16,bf16,bf16s,fp32] [--repeats R]
    python tools/xent_bench.py train [--mode fused|hooks] [--steps K] [--warmup W]

``eval`` times the MLP evaluate launch alone (CUDA events, ms per launch), cross-entropy against the
squared error on the same weights and batch: at the north-star body with a 256-class head
(P = 4096, [128, 512, 512, 512, 512, 256], B = 256) in each precision mode, and in fp32 at an
MNIST-shaped [784, 256, 10] (P = 4096, B = 256).  ``train`` times ``ES.train`` generations of a
cross-entropy classifier at the north-star body through the public API: fused (a DeviceAgent with
``loss="cross_entropy"``) or hooks mode (a host agent with the same rollout).  The card name and power
limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NORTH_256 = [128, 512, 512, 512, 512, 256]
MNIST = [784, 256, 10]
XENT = 1 << 16                     # ESTK_LOSS_XENT


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def emit(**kw):
    print(json.dumps(kw), flush=True)


def eval_times(args):
    from estorch_b200.backend import CudaBackend
    be = CudaBackend(torch.device("cuda", 0))
    pairs, B = 2048, 256
    table = be.alloc(1 << 28)
    be.fill_noise_table(table, 42)
    tb16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, tb16) == 0
    tbb = be.alloc(table.numel(), dtype=torch.bfloat16)
    be.shadow_bf16(table, tbb)
    gpu = card()
    cases = [(NORTH_256, m) for m in args.modes.split(",")] + [(MNIST, "fp32")]
    torch.manual_seed(0)
    setup = {}
    for dims, _ in cases:
        key = tuple(dims)
        if key in setup:
            continue
        n = sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))
        offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
        be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
        theta = torch.randn(n, device=be.device) * 0.05
        th16 = None
        if dims == NORTH_256:                      # the bf16 shadow of theta ("bf16s" only)
            th16 = be.alloc(n, dtype=torch.bfloat16)
            be.shadow_bf16(theta, th16)
        obs = torch.randn(B, dims[0], device=be.device)
        tgt = torch.nn.functional.one_hot(torch.randint(0, dims[-1], (B,), device=be.device), dims[-1]).float()
        setup[key] = (offs, order, theta, th16, obs, tgt)
    ret = be.zeros(2 * pairs)
    for rep in range(args.repeats):
        for dims, mode in cases:
            offs, order, theta, th16, obs, tgt = setup[tuple(dims)]
            for loss, code in (("mse", 0), ("cross_entropy", XENT)):
                kw = {"table16": tb16} if mode == "f16" else {"theta16": th16, "table16": tbb} if mode == "bf16s" else {}
                if code:
                    kw["act"] = code

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
                emit(what="eval", dims=dims, loss=loss, mode=mode, ms=round(e0.elapsed_time(e1) / args.iters, 4),
                     repeat=rep, checksum=float(ret.double().sum()), gpu=gpu)


class Policy(torch.nn.Module):
    def __init__(self, dims):
        super().__init__()
        layers = []
        for i in range(len(dims) - 1):
            layers.append(torch.nn.Linear(dims[i], dims[i + 1]))
            if i + 2 < len(dims):
                layers.append(torch.nn.ReLU())
        self.net = torch.nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


class HostAgent:
    """The same rollout as DeviceAgent(loss="cross_entropy"), as a plain agent: hooks mode."""
    def __init__(self, obs, target):
        import estorch_b200 as E
        self.inner = E.DeviceAgent(obs, target, loss="cross_entropy")

    def rollout(self, policy):
        return self.inner.rollout(policy)


def train_rate(args):
    import estorch_b200 as E
    dims = NORTH_256
    g = torch.Generator().manual_seed(1234)
    obs = torch.randn(256, dims[0], generator=g)
    tgt = torch.nn.functional.one_hot(torch.randint(0, dims[-1], (256,), generator=g), dims[-1]).float()
    torch.manual_seed(0)
    fused = args.mode == "fused"
    es = E.ES(Policy, E.DeviceAgent if fused else HostAgent, torch.optim.Adam, population_size=args.population,
              sigma=0.02, policy_kwargs={"dims": dims},
              agent_kwargs=dict(obs=obs, target=tgt, **({"loss": "cross_entropy"} if fused else {})),
              optimizer_kwargs={"lr": 0.01}, device=torch.device("cuda", 0), log_interval=10 ** 9)
    es.log = lambda: None
    if args.warmup:
        es.train(n_steps=args.warmup)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    es.train(n_steps=args.steps)
    torch.cuda.synchronize()
    s = time.perf_counter() - t0
    emit(what="train", mode=args.mode, dims=dims, population=args.population, fused=bool(es._fused),
         precision=es._precision, steps=args.steps, seconds=round(s, 4), generations_per_s=round(args.steps / s, 4),
         episode_reward=float(es.episode_reward), gpu=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["eval", "train"])
    ap.add_argument("--modes", default="f16,bf16,bf16s,fp32")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--mode", default="fused", choices=["fused", "hooks"])
    ap.add_argument("--population", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    eval_times(args) if args.what == "eval" else train_rate(args)


if __name__ == "__main__":
    main()
