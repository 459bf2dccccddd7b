"""The F16 arithmetic for every MLP shape (ESTK_PREC_F16_ANY) against fp32 (one JSON line per measurement).

    python tools/f16_any_bench.py eval     [--iters N] [--warmup W]
    python tools/f16_any_bench.py train    [--steps K] [--warmup W]
    python tools/f16_any_bench.py accuracy [--members M]

``eval`` times estk_eval_mlp per case with precision "f16_any" and "fp32", alternated (CUDA events over N
launches after W warm-up launches), and reports ms per launch and the rate 2 * n * B * P / t.  The kernels
of every case are read from one torch.profiler session before the timing.  ``train`` times ES.train
generations of the [3072,512,10] cross-entropy classifier at P = 4096, B = 256 with eval_precision "f16"
(the streamed tensor-core kernel) and "fp32", alternated.  ``accuracy`` compares the returns of M members of
the [3072,512,10] and [784,256,10] classifiers against the CPU fp32 forward (max-norm relative error).
The card's name, power limit and max SM clock are printed with the numbers.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
XENT = 1 << 16                     # ESTK_LOSS_XENT
CIFAR = [3072, 512, 10]
# (dims, B, P, loss code)
CASES = [([784, 256, 10], 256, 4096, 0), ([784, 256, 10], 1024, 4096, 0), (CIFAR, 256, 4096, XENT),
         ([1088, 1088, 1088, 32], 256, 4096, 0), ([64, 4096, 4096, 8], 256, 512, 0),
         ([784, 128, 10], 60000, 256, 0), ([4, 64, 64, 2], 256, 4096, 0)]
PRECISIONS = ("f16_any", "fp32")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def emit(**kw):
    print(json.dumps(kw), flush=True)


def setup(be, table, table16, dims, B, P, code, precision, seed=0):
    """(run, ret, n): one evaluate launch of the case on seeded inputs."""
    g = torch.Generator(device=be.device).manual_seed(seed)
    pairs = P // 2
    n = sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))
    offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
    theta = torch.randn(n, device=be.device, generator=g) / dims[0] ** 0.5
    obs = torch.randn(B, dims[0], device=be.device, generator=g)
    if code:
        cls = torch.randint(0, dims[-1], (B,), device=be.device, generator=g)
        tgt = torch.nn.functional.one_hot(cls, dims[-1]).float()
    else:
        tgt = torch.randn(B, dims[-1], device=be.device, generator=g)
    ret = be.zeros(2 * pairs)
    kw = {"table16": table16} if precision != "fp32" else {}

    def run():
        be.eval_mlp(dims, theta, table, offs, order, pairs, 0.02, obs, tgt, ret[:pairs], ret[pairs:], act=code,
                    precision=precision, **kw)
    return run, ret, n, (theta, offs, obs, tgt)


def kernel_names(be, table, table16):
    """The kernels of every (case, precision), in one profiling session: the process's first."""
    from torch.profiler import ProfilerActivity, profile
    keys = [(i, p) for i in range(len(CASES)) for p in PRECISIONS]
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i, p in keys:
            run = setup(be, table, table16, *CASES[i], p)[0]
            run()
            torch.cuda.synchronize()
            torch.ones(1, device=be.device).mul_(2.0)      # a separator kernel between cases
            torch.cuda.synchronize()
    found = sorted((e.time_range.start, e.name) for e in prof.events()
                   if e.device_type == torch.autograd.DeviceType.CUDA)
    groups, cur = [], []
    for _, name in found:
        if "eval_mlp" in name or "split_obs" in name:
            cur.append(re.search(r"\w+_kernel(<[^>]*>)?", name).group(0))
        elif cur:
            groups.append("+".join(cur))
            cur = []
    return dict(zip(keys, groups)) if len(groups) == len(keys) else {k: "not recorded" for k in keys}


def eval_times(args):
    from estorch_b200.backend import CudaBackend
    be = CudaBackend(torch.device("cuda", 0))
    gpu = card()
    table = be.alloc(1 << 26)
    be.fill_noise_table(table, 42)
    table16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, table16) == 0
    names = kernel_names(be, table, table16)
    for i, (dims, B, P, code) in enumerate(CASES):
        runs = {p: setup(be, table, table16, dims, B, P, code, p) for p in PRECISIONS}
        ms = {p: [] for p in PRECISIONS}
        for p in PRECISIONS:
            for _ in range(args.warmup):
                runs[p][0]()
        torch.cuda.synchronize()
        for rep in range(args.reps):                       # alternated: f16_any, fp32, f16_any, ...
            for p in PRECISIONS:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    runs[p][0]()
                e1.record()
                torch.cuda.synchronize()
                ms[p].append(e0.elapsed_time(e1) / args.iters)
        n = runs["fp32"][2]
        ra, rf = runs["f16_any"][1].cpu().numpy(), runs["fp32"][1].cpu().numpy()
        for p in PRECISIONS:
            t = min(ms[p])
            emit(what="eval", precision=p, dims=dims, B=B, P=P, loss="cross_entropy" if code else "mse",
                 ms=round(t, 3), ms_all=[round(x, 3) for x in ms[p]], tflops=round(2.0 * n * B * P / (t * 1e-3) / 1e12, 2),
                 iters=args.iters, kernel=names[(i, p)], gpu=gpu)
        emit(what="eval_ratio", dims=dims, B=B, P=P, fp32_over_f16_any=round(min(ms["fp32"]) / min(ms["f16_any"]), 2),
             returns_rel_vs_fp32=float(np.abs(ra - rf).max() / np.abs(rf).max()), gpu=gpu)
        del runs


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


def train_rate(args):
    import estorch_b200 as E
    dims = CIFAR
    g = torch.Generator().manual_seed(1234)
    obs = torch.randn(256, dims[0], generator=g)
    tgt = torch.nn.functional.one_hot(torch.randint(0, dims[-1], (256,), generator=g), dims[-1]).float()
    ess = {}
    for p in ("f16", "fp32"):
        torch.manual_seed(0)
        es = E.ES(Policy, E.DeviceAgent, torch.optim.Adam, population_size=args.population, sigma=0.02,
                  policy_kwargs={"dims": dims}, agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy"),
                  optimizer_kwargs={"lr": 0.01}, device=torch.device("cuda", 0), log_interval=10 ** 9,
                  eval_precision=p)
        es.log = lambda: None
        es.train(n_steps=args.warmup)
        ess[p] = es
    rates = {p: [] for p in ess}
    for rep in range(args.reps):
        for p, es in ess.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            es.train(n_steps=args.steps)
            torch.cuda.synchronize()
            rates[p].append(args.steps / (time.perf_counter() - t0))
    for p, es in ess.items():
        emit(what="train", eval_precision=p, precision=es._precision, dims=dims, population=args.population,
             fused=bool(es._fused), steps=args.steps, generations_per_s=round(max(rates[p]), 3),
             all=[round(r, 3) for r in rates[p]], gpu=card())


def accuracy(args):
    from estorch_b200.backend import CudaBackend
    from oracle import es_oracle as orc
    be = CudaBackend(torch.device("cuda", 0))
    table = be.alloc(1 << 24)
    be.fill_noise_table(table, 42)
    table16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, table16) == 0
    tb = table.cpu().numpy()
    for dims in (CIFAR, [784, 256, 10]):
        run, ret, n, (theta, offs, obs, tgt) = setup(be, table, table16, dims, 256, args.members, XENT, "f16_any")
        run()
        torch.cuda.synchronize()
        got = ret.cpu().numpy()
        pop, _ = orc.sample_population(theta.cpu().numpy(), tb, offs.cpu().numpy(), 0.02)
        x, t = obs.cpu().numpy(), tgt.cpu().numpy().astype(np.float64)
        want = np.empty(len(pop), np.float32)
        for i, row in enumerate(pop):
            y = orc.mlp_forward(row, dims, x).astype(np.float64)
            m = y.max(axis=1, keepdims=True)
            lse = m[:, 0] + np.log(np.exp(y - m).sum(axis=1))
            want[i] = -(lse * t.sum(axis=1) - (t * y).sum(axis=1)).sum() / y.shape[0]
        emit(what="accuracy", dims=dims, B=256, members=len(pop), loss="cross_entropy",
             rel_vs_cpu_fp32=float(np.abs(got - want).max() / np.abs(want).max()), gpu=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["eval", "train", "accuracy"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--population", type=int, default=4096)
    ap.add_argument("--members", type=int, default=512)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    {"eval": eval_times, "train": train_rate, "accuracy": accuracy}[args.what](args)


if __name__ == "__main__":
    main()
