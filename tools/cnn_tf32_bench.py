#!/usr/bin/env python
"""Measure the TF32 convolutional evaluate (estk_eval_cnn_tf32) against the fp32 one (estk_eval_mlp with n_conv) on
tools/cnn_bench.py's three shapes: (a) an MNIST-shape classifier, (b) the Atari network without VirtualBatchNorm,
(c) a MinAtar-shape network, at B and P of DESIGN §9.

Per shape: the fp32 and tf32 evaluate launches alternated in one process (CUDA events, warmed up; the median of
the rounds), the achieved TFLOP/s from the shape's multiply-adds against the H100 SXM data-sheet 495 TFLOP/s dense
TF32, the returns' max-norm relative distance between the two modes, and the torch alternative (materialised rows,
grouped F.conv2d, baddbmm) with torch.backends.cudnn.allow_tf32 (and cuda.matmul.allow_tf32) False and True.
Then generations/s of fused ES.train in "tf32" and in "fp32".  Prints one JSON line per row, the first with the
card and its power limit, and writes them to --out."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from cnn_bench import SHAPES, _time, macs, pack, policy_class, torch_eval  # noqa: E402
from estorch_b200 import ES, DeviceAgent, _capi  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402
from estorch_b200.policy_spec import CNNSpec  # noqa: E402

PEAK_TF32 = 495e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def kernel_rows(be, rounds, reps32, reps):
    out = []
    for name, (shape, convs, linears, xent, B, pops) in SHAPES.items():
        dims, n_conv = pack(shape, convs, linears), len(convs)
        code = n_conv << 24 | (_capi.ESTK_LOSS_XENT if xent else 0)
        n = CNNSpec(shape, tuple(convs), tuple(linears)).n_parameters
        g = torch.Generator().manual_seed(0)
        obs = torch.rand(B, *shape, generator=g).to(be.device)
        tgt = torch.rand(B, linears[-1], generator=g).to(be.device)
        theta = (torch.randn(n, generator=g) * 0.05).to(be.device)
        table = be.alloc((n + 31) // 32 * 32 + (1 << 22))
        be.fill_noise_table(table, 1)
        P = pops[0]
        pairs = P // 2
        offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
        be.make_offsets(3, None, 0, 0, pairs, table.numel(), n, offsets, order)
        rets = {m: be.zeros(P) for m in ("fp32", "tf32")}

        def run(mode):
            r = rets[mode]
            be.eval_cnn(dims, theta, table, offsets, order, pairs, 0.05, obs, tgt, r[:pairs], r[pairs:], act=code,
                        precision=mode)
        times = {"fp32": [], "tf32": []}
        for _ in range(rounds):
            for mode, k in (("fp32", reps32), ("tf32", reps)):
                times[mode].append(_time(lambda: run(mode), k))
        med = {m: sorted(v)[len(v) // 2] for m, v in times.items()}
        flops = 2.0 * macs(shape, convs, linears) * B * P
        r32, rtf = rets["fp32"].double(), rets["tf32"].double()
        row = dict(kind="evaluate", shape=name, B=B, P=P, fp32_ms=round(med["fp32"] * 1e3, 3),
                   tf32_ms=round(med["tf32"] * 1e3, 3), speedup=round(med["fp32"] / med["tf32"], 2),
                   tf32_spread_ms=[round(min(times["tf32"]) * 1e3, 3), round(max(times["tf32"]) * 1e3, 3)],
                   tf32_tflops=round(flops / med["tf32"] / 1e12, 2),
                   tf32_of_peak=round(flops / med["tf32"] / PEAK_TF32, 4),
                   returns_rel=float((rtf - r32).abs().max() / r32.abs().max()))
        rows = be.alloc(P, n)
        c1 = convs[0]
        act1 = c1[0] * ((shape[1] + 2 * c1[3] - c1[1]) // c1[2] + 1) * ((shape[2] + 2 * c1[3] - c1[1]) // c1[2] + 1)
        chunk = max(1, min(P, (1 << 30) // (4 * B * act1)))
        for allow in (False, True):
            torch.backends.cudnn.allow_tf32 = allow
            torch.backends.cuda.matmul.allow_tf32 = allow
            tt = _time(lambda: torch_eval(be, convs, linears, theta, table, offsets, pairs, obs, tgt, rows, chunk),
                       max(2, reps // 5))
            row[f"torch_allow_tf32_{allow}_ms"] = round(tt * 1e3, 3)
        torch.backends.cudnn.allow_tf32 = True
        torch.backends.cuda.matmul.allow_tf32 = False
        del rows
        torch.cuda.empty_cache()
        print(json.dumps(row), flush=True)
        out.append(row)
    return out


def train_rows(be, gens):
    out = []
    for name, (shape, convs, linears, xent, B, pops) in SHAPES.items():
        g = torch.Generator().manual_seed(0)
        obs = torch.rand(B, *shape, generator=g)
        tgt = torch.rand(B, linears[-1], generator=g)
        row = dict(kind="train", shape=name, P=pops[0], B=B)
        for mode in ("fp32", "tf32"):
            torch.manual_seed(0)
            es = ES(policy_class(shape, convs, linears), DeviceAgent, torch.optim.Adam, population_size=pops[0],
                    sigma=0.05, agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy" if xent else "mse"),
                    optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 24, eval_precision=mode, _backend=be)
            assert es._fused and es._precision == mode
            es.log = lambda: None
            es.train(n_steps=2)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            es.train(n_steps=gens)
            torch.cuda.synchronize()
            row[f"{mode}_gens_per_s"] = round(gens / (time.perf_counter() - t0), 3)
        print(json.dumps(row), flush=True)
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps32", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--gens", type=int, default=5)
    ap.add_argument("--no-train", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("cnn_tf32_bench: needs a CUDA GPU")
    head = dict(kind="card", card=card())
    print(json.dumps(head), flush=True)
    be = CudaBackend()
    rows = [head] + kernel_rows(be, a.rounds, a.reps32, a.reps)
    if not a.no_train:
        rows += train_rows(be, a.gens)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
