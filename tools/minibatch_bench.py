#!/usr/bin/env python
"""Measure minibatches drawn on the device (estk_sample_batch, estk_batch.cu).

(a) The sampler alone: B = 256 rows of 784 and of 3072 floats (and their 10-float targets) gathered from an
    N = 60,000-row dataset, CUDA events around many back-to-back launches, in us per launch and the GB/s of the
    bytes it reads and writes.
(b) Generations/s of ``ES.train`` for a [784, 256, 10] cross-entropy MLP at P = 4096 in three forms of the same
    B = 256: minibatches drawn on the device (``batch_size=256`` over N = 60,000 rows), the ``next_batch`` host
    hook returning fresh pinned tensors of the same rows every generation (kept alive, so that their addresses do
    not repeat), and one fixed batch.  The three
    alternate within every repetition.

Prints one JSON line per row, the first with the card and its power limit, and writes them to --out."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from estorch_b200 import ES, DeviceAgent, batch_indices  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def sampler(be, n, row, trow, b, launches):
    g = torch.Generator().manual_seed(row)
    obs = torch.randn(n, row, generator=g).to(be.device)
    tgt = torch.randn(n, trow, generator=g).to(be.device)
    dst, tdst = be.alloc(b, row), be.alloc(b, trow)
    for i in range(50):
        be.sample_batch(1, None, i, obs, dst, tgt, tdst)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(launches):
        be.sample_batch(1, None, i, obs, dst, tgt, tdst)
    t1.record()
    torch.cuda.synchronize()
    us = t0.elapsed_time(t1) * 1e3 / launches
    moved = 2 * b * (row + trow) * 4
    return {"kind": "sampler", "N": n, "B": b, "row_floats": row, "target_floats": trow, "us_per_launch": us,
            "bytes_read_and_written": moved, "GB_per_s": moved / us / 1e3, "launches": launches}


class MLP(nn.Module):
    def __init__(self):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(784, 256), nn.ReLU(), nn.Linear(256, 10))

    def forward(self, x):
        return self.net(x)


def make(mode, x, y, b, P):
    if mode == "device_sampling":
        agent, akw = DeviceAgent, dict(obs=x, target=y, loss="cross_entropy", batch_size=b)
    elif mode == "fixed_batch":
        agent, akw = DeviceAgent, dict(obs=x[:b], target=y[:b], loss="cross_entropy")
    else:
        class Uploading(DeviceAgent):
            handed = []

            def next_batch(self, step):
                # fresh pinned tensors, kept alive: a recycled pinned block would repeat the graph key, and the
                # generation that captures it would capture the upload from host memory
                idx = torch.from_numpy(batch_indices(0, step, x.shape[0], b))
                self.handed.append((x[idx].pin_memory(), y[idx].pin_memory()))
                return self.handed[-1]
        i0 = torch.from_numpy(batch_indices(0, 0, x.shape[0], b))
        agent, akw = Uploading, dict(obs=x[i0], target=y[i0], loss="cross_entropy")
    torch.manual_seed(0)
    es = ES(MLP, agent, torch.optim.Adam, population_size=P, sigma=0.02, agent_kwargs=akw,
            optimizer_kwargs={"lr": 0.01})
    es.log = lambda: None
    return es


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=60000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--population", type=int, default=4096)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--gens", type=int, default=50, help="generations per timed train() call")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    lines = [dict(card(), command=" ".join(sys.argv))]
    print(json.dumps(lines[-1]), flush=True)
    be = CudaBackend(torch.device("cuda", 0))
    for row in (784, 3072):
        lines.append(sampler(be, a.rows, row, 10, a.batch, a.launches))
        print(json.dumps(lines[-1]), flush=True)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(a.rows, 784, generator=g)
    y = nn.functional.one_hot(torch.randint(0, 10, (a.rows,), generator=g), 10).float()
    modes = ("device_sampling", "next_batch_upload", "fixed_batch")
    runs = {m: make(m, x, y, a.batch, a.population) for m in modes}
    for es in runs.values():
        es.train(n_steps=10)                # captures the graphs where they apply
    torch.cuda.synchronize()
    rates = {m: [] for m in modes}
    for _ in range(a.reps):
        for m in modes:
            es = runs[m]
            torch.cuda.synchronize()
            t = time.perf_counter()
            es.train(n_steps=a.gens)
            torch.cuda.synchronize()
            rates[m].append(a.gens / (time.perf_counter() - t))
    for m in modes:
        r = sorted(rates[m])
        lines.append({"kind": "train", "mode": m, "dims": [784, 256, 10], "loss": "cross_entropy",
                      "P": a.population, "B": a.batch, "N": a.rows if m != "fixed_batch" else a.batch,
                      "precision": runs[m]._precision, "graphs": sum(isinstance(v, tuple) for v in
                                                                     runs[m].__dict__.get("_graphs", {}).values()),
                      "gens_per_s_median": r[len(r) // 2], "gens_per_s_min": r[0], "gens_per_s_max": r[-1]})
        print(json.dumps(lines[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
