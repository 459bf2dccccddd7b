"""The streamed fp32 evaluate (eval_mlp_wide_kernel) at the shapes it serves (one JSON line per measurement).

    python tools/wide_bench.py eval  [--iters N] [--warmup W]
    python tools/wide_bench.py train [--mode fused|hooks] [--steps K] [--warmup W]

``eval`` times estk_eval_mlp with ESTK_PREC_FP32 (CUDA events over N launches after W warm-up launches) and
reports ms per launch and the achieved rate 2 * n * B * P / t, for: [1024,1024,1024,32], the widest shape
the shared-memory kernel runs, against [1088,1088,1088,32] just past it; [3072,512,10] cross-entropy;
[784,256,10] at B = 1024 and B = 60,000; [64,4096,4096,8].  Every line names the kernel that ran (read
from torch.profiler in one session before the timing).  ``train`` times ES.train generations of the [3072,512,10]
cross-entropy classifier at P = 4096, B = 256: fused, or hooks mode (a host agent wrapping
DeviceAgent.rollout).  The card name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
XENT = 1 << 16                     # ESTK_LOSS_XENT
CIFAR = [3072, 512, 10]
# (dims, B, P, loss code)
CASES = [([1024, 1024, 1024, 32], 256, 4096, 0), ([1088, 1088, 1088, 32], 256, 4096, 0),
         (CIFAR, 256, 4096, XENT),
         ([784, 256, 10], 1024, 4096, 0), ([784, 256, 10], 60000, 256, 0),
         ([64, 4096, 4096, 8], 256, 512, 0)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def emit(**kw):
    print(json.dumps(kw), flush=True)


def setup(be, table, dims, B, P, code):
    """(run, ret, n): one evaluate launch of the case on fresh seeded inputs."""
    pairs = P // 2
    n = sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))
    offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
    theta = torch.randn(n, device=be.device) / dims[0] ** 0.5
    obs = torch.randn(B, dims[0], device=be.device)
    if code:
        tgt = torch.nn.functional.one_hot(torch.randint(0, dims[-1], (B,), device=be.device), dims[-1]).float()
    else:
        tgt = torch.randn(B, dims[-1], device=be.device)
    ret = be.zeros(2 * pairs)

    def run():
        be.eval_mlp(dims, theta, table, offs, order, pairs, 0.02, obs, tgt, ret[:pairs], ret[pairs:], act=code)
    return run, ret, n


def kernel_names(be, table):
    """The evaluate kernel of every case, in one profiling session: the process's first (a later session,
    after CUPTI was torn down at the end of an earlier one, may record no GPU activity)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for case in CASES:
            run, _, _ = setup(be, table, *case)
            run()
            torch.cuda.synchronize()
            del run
    found = sorted((e.time_range.start, m.group(0)) for e in prof.events()
                   if e.device_type == torch.autograd.DeviceType.CUDA
                   for m in [re.search(r"eval_mlp\w*<[^>]*>", e.name)] if m)
    names = [name for _, name in found]
    return names if len(names) == len(CASES) else ["not recorded"] * len(CASES)


def eval_times(args):
    from estorch_b200.backend import CudaBackend
    be = CudaBackend(torch.device("cuda", 0))
    gpu = card()
    table = be.alloc(1 << 26)
    be.fill_noise_table(table, 42)
    torch.manual_seed(0)
    names = kernel_names(be, table)
    torch.manual_seed(0)
    for (dims, B, P, code), kernel in zip(CASES, names):
        run, ret, n = setup(be, table, dims, B, P, code)
        for _ in range(args.warmup):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        emit(what="eval", dims=dims, B=B, P=P, loss="cross_entropy" if code else "mse", ms=round(ms, 3),
             tflops=round(2.0 * n * B * P / (ms * 1e-3) / 1e12, 3), iters=args.iters, kernel=kernel,
             checksum=float(ret.double().sum()), gpu=gpu)
        del run, ret


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
    dims = CIFAR
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
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--mode", default="fused", choices=["fused", "hooks"])
    ap.add_argument("--population", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    eval_times(args) if args.what == "eval" else train_rate(args)


if __name__ == "__main__":
    main()
