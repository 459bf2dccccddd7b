"""Cost of the accuracy objective against the cross-entropy (one JSON line per measurement).

    python tools/accuracy_bench.py eval  [--iters N] [--repeats R]
    python tools/accuracy_bench.py train [--steps K] [--warmup W] [--hooks-steps H]

``eval`` times the evaluate launch alone with CUDA events, ms per launch, alternating loss="accuracy" and
loss="cross_entropy" on the same weights, noise and batch (P = 4096, B = 256): [784, 256, 10] in fp32 and in
f16_any, the north-star body with a 256-class head ([128, 512, 512, 512, 512, 256]) in f16, and the "a_mnist" CNN of
tools/cnn_bench.py in fp32.  ``train`` times ``ES.train`` generations of the [784, 256, 10] classifier with the
accuracy as the return: fused (``DeviceAgent(loss="accuracy")``) against hooks mode (a host agent with the same
rollout).  The card name and power limit are read in the same run and printed with every line.
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
XENT, ACC = 1 << 16, 6 << 16       # ESTK_LOSS_XENT, ESTK_LOSS_ACCURACY
MNIST = [784, 256, 10]
NORTH_256 = [128, 512, 512, 512, 512, 256]
CNN = ((1, 28, 28), ((16, 5, 2, 2), (32, 5, 2, 2)), (10,))


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
    from estorch_b200.policy_spec import CNNSpec
    be = CudaBackend(torch.device("cuda", 0))
    gpu = card()
    pairs, B = 2048, 256
    table = be.alloc(1 << 26)
    be.fill_noise_table(table, 42)
    tb16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, tb16) == 0
    cnn = CNNSpec(*CNN)
    cases = [("mlp", MNIST, "fp32"), ("mlp", MNIST, "f16_any"), ("mlp", NORTH_256, "f16"), ("cnn", cnn.dims, "fp32")]
    g = torch.Generator().manual_seed(0)
    ret = be.zeros(2 * pairs)
    runs = []
    for kind, dims, mode in cases:
        n = cnn.n_parameters if kind == "cnn" else sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))
        offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
        be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
        theta = (torch.randn(n, generator=g) * 0.05).to(be.device)
        obs = torch.randn(B, *(CNN[0] if kind == "cnn" else (dims[0],)), generator=g).to(be.device)
        C = CNN[2][-1] if kind == "cnn" else dims[-1]
        tgt = torch.nn.functional.one_hot(torch.randint(0, C, (B,), generator=g), C).float().to(be.device)
        for loss, code in (("accuracy", ACC), ("cross_entropy", XENT)):
            if kind == "cnn":
                def run(code=code, dims=dims, theta=theta, offs=offs, order=order, obs=obs, tgt=tgt):
                    be.eval_cnn(dims, theta, table, offs, order, pairs, 0.02, obs, tgt, ret[:pairs], ret[pairs:],
                                act=len(CNN[1]) << 24 | code)
            else:
                kw = {"table16": tb16} if mode in ("f16", "f16_any") else {}

                def run(code=code, dims=dims, theta=theta, offs=offs, order=order, obs=obs, tgt=tgt, mode=mode, kw=kw):
                    be.eval_mlp(dims, theta, table, offs, order, pairs, 0.02, obs, tgt, ret[:pairs], ret[pairs:],
                                precision=mode, act=code, **kw)
            runs.append((kind, dims if kind == "mlp" else "a_mnist", mode, loss, run))
    for _, _, _, _, run in runs:              # warm every shape up before any timed window
        for _ in range(3):
            run()
    torch.cuda.synchronize()
    for rep in range(args.repeats):
        for kind, dims, mode, loss, run in runs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                run()
            e1.record()
            torch.cuda.synchronize()
            emit(what="eval", kind=kind, dims=dims, mode=mode, loss=loss, P=2 * pairs, B=B,
                 ms=round(e0.elapsed_time(e1) / args.iters, 4), repeat=rep, gpu=gpu)


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
    """The same rollout as DeviceAgent(loss="accuracy"), as a plain agent: hooks mode."""
    def __init__(self, obs, target):
        import estorch_b200 as E
        self.inner = E.DeviceAgent(obs, target, loss="accuracy")

    def rollout(self, policy):
        return self.inner.rollout(policy)


def train_rate(args):
    import estorch_b200 as E
    gpu = card()
    g = torch.Generator().manual_seed(1234)
    obs = torch.randn(256, MNIST[0], generator=g)
    tgt = torch.nn.functional.one_hot(torch.randint(0, MNIST[-1], (256,), generator=g), MNIST[-1]).float()
    for mode, steps in (("fused", args.steps), ("hooks", args.hooks_steps)):
        torch.manual_seed(0)
        fused = mode == "fused"
        es = E.ES(Policy, E.DeviceAgent if fused else HostAgent, torch.optim.Adam, population_size=args.population,
                  sigma=0.02, policy_kwargs={"dims": MNIST},
                  agent_kwargs=dict(obs=obs, target=tgt, **({"loss": "accuracy"} if fused else {})),
                  optimizer_kwargs={"lr": 0.01}, device=torch.device("cuda", 0), log_interval=10 ** 9)
        es.log = lambda: None
        es.train(n_steps=args.warmup if fused else 1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        es.train(n_steps=steps)
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        emit(what="train", mode=mode, dims=MNIST, population=args.population, fused=bool(es._fused),
             precision=es._precision, steps=steps, seconds=round(s, 4), generations_per_s=round(steps / s, 4),
             episode_reward=float(es.episode_reward), gpu=gpu)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=["eval", "train"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--population", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--hooks-steps", type=int, default=1)
    args = ap.parse_args()
    eval_times(args) if args.what == "eval" else train_rate(args)


if __name__ == "__main__":
    main()
