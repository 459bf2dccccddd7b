"""Evaluate time and training rate of MLP policies by activation (one JSON line per measurement).

    python tools/act_bench.py eval  [--acts relu,tanh,relu+tanh,tanh+tanh] [--modes f16,bf16,bf16s,fp32]
    python tools/act_bench.py train --shape cartpole|north_star --hidden tanh [--output tanh] [--steps K] [--warmup W]

``eval`` times the MLP evaluate launch alone at the north star (P = 4096, n = 1,001,760, B = 256; CUDA
events, ms per launch) for each activation (hidden[+output]) and precision mode.  ``train`` times
``ES.train`` generations of a policy with the given activations through the public API (fused when
the engine recognises the policy, hooks mode otherwise).  Activation codes other than ReLU are only
passed to libraries that define them, so the same script times an older build (ESTK_LIBRARY, or
the script run from an older tree) on ReLU.  The card name and power limit are printed with the numbers.
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
MLP_1M = [128, 512, 512, 512, 512, 288]
SHAPES = {"north_star": MLP_1M, "cartpole": [4, 64, 64, 2]}
ACT_CODES = {"relu": 0, "tanh": 1, "relu+tanh": 1 << 8, "tanh+tanh": 1 | 1 << 8}


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
                if ACT_CODES[a]:
                    kw["act"] = ACT_CODES[a]

                def run():
                    be.eval_mlp(dims, theta, table, offs, order, pairs, 0.02, obs, tgt, ret[:pairs], ret[pairs:],
                                precision=mode, **kw)
                try:
                    for _ in range(3):
                        run()
                except (RuntimeError, TypeError) as e:
                    emit(what="eval", act=a, mode=mode, error=str(e)[:120])
                    continue
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    run()
                e1.record()
                torch.cuda.synchronize()
                emit(what="eval", act=a, mode=mode, ms=round(e0.elapsed_time(e1) / args.iters, 4), repeat=rep,
                     checksum=float(ret.double().sum()), library=os.environ.get("ESTK_LIBRARY", "tree"), gpu=gpu)


class Policy(torch.nn.Module):
    def __init__(self, dims, hidden="tanh", output="identity"):
        super().__init__()
        act = {"relu": torch.nn.ReLU, "tanh": torch.nn.Tanh}
        layers = []
        for i in range(len(dims) - 1):
            layers.append(torch.nn.Linear(dims[i], dims[i + 1]))
            if i + 2 < len(dims):
                layers.append(act[hidden]())
        if output == "tanh":
            layers.append(torch.nn.Tanh())
        self.net = torch.nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


def train_rate(args):
    import estorch_b200 as E
    dims = SHAPES[args.shape]
    g = torch.Generator().manual_seed(1234)
    obs, tgt = torch.randn(256, dims[0], generator=g), torch.rand(256, dims[-1], generator=g) * 1.8 - 0.9
    torch.manual_seed(0)
    es = E.ES(Policy, E.DeviceAgent, torch.optim.Adam, population_size=args.population, sigma=0.02,
              policy_kwargs={"dims": dims, "hidden": args.hidden, "output": args.output},
              agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01},
              log_interval=10 ** 9)
    es.log = lambda: None
    if args.warmup:
        es.train(n_steps=args.warmup)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    es.train(n_steps=args.steps)
    torch.cuda.synchronize()
    s = time.perf_counter() - t0
    emit(what="train", shape=args.shape, hidden=args.hidden, output=args.output, population=args.population,
         fused=bool(es._fused), precision=es._precision, steps=args.steps, seconds=round(s, 4),
         generations_per_s=round(args.steps / s, 4), episode_reward=float(es.episode_reward), gpu=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["eval", "train"])
    ap.add_argument("--acts", default="relu,tanh,relu+tanh,tanh+tanh")
    ap.add_argument("--modes", default="f16,bf16,bf16s,fp32")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--shape", default="cartpole", choices=sorted(SHAPES))
    ap.add_argument("--hidden", default="tanh", choices=["relu", "tanh"])
    ap.add_argument("--output", default="identity", choices=["identity", "tanh"])
    ap.add_argument("--population", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    eval_times(args) if args.what == "eval" else train_rate(args)


if __name__ == "__main__":
    main()
