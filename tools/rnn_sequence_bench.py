#!/usr/bin/env python
"""Time the recurrent sequence evaluate (estk_eval_mlp with a cell code and a return) on one GPU.

For GRU / LSTM with H in {32, 64, 128, 256}, in 8, out 4, T 32, B 64 and P 4096 (2048 antithetic pairs):
  seq_ms    one sequence-evaluate launch (CUDA events, mean over the timed launches);
  steps_ms  the same work composed from T ESTK_ACTIONS step launches (every member's [x_t | state] rows
            built with torch) plus the squared error in torch;
and ``ES.train`` generations/s for a GRU H = 64 SequenceAgent at P = 256: fused mode against hooks mode (one
torch rollout per member on the GPU).  Prints one JSON line per row, the first with the card, its power limit and the
library (ESTK_LIBRARY selects a triage build of a kernel variant), and writes them to --out."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from estorch_b200 import ES, SequenceAgent, _capi  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402
from _rnn_oracle import CELL_GRU, CELL_LSTM, param_count, policy_class  # noqa: E402


def _time(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernel_rows(be, reps):
    rows = []
    i, o, T, B, P = 8, 4, 32, 64, 4096
    pairs = P // 2
    g = torch.Generator().manual_seed(0)
    obs = torch.randn(B, T, i, generator=g).to(be.device)
    tgt = (torch.rand(B, T, o, generator=g) * 1.6 - 0.8).to(be.device)
    for cell, code in (("gru", CELL_GRU), ("lstm", CELL_LSTM)):
        for H in (32, 64, 128, 256):
            dims = (i, H, o)
            n = param_count(cell, dims)
            theta = ((torch.rand(n, generator=g) * 2 - 1) / H ** 0.5).to(be.device)
            table = be.alloc((n + 31) // 32 * 32 + 32 * 8192)
            be.fill_noise_table(table, 3)
            offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
            be.make_offsets(1, None, 0, 0, pairs, table.numel(), n, offsets, order)
            ret = be.zeros(P)

            def seq():
                be.eval_rnn_seq(dims, theta, table, offsets, order, pairs, 0.05, obs, tgt, ret[:pairs], ret[pairs:],
                                act=code)
            S = H if cell == "gru" else 2 * H

            def steps():
                state = torch.zeros(P, B, S, device=be.device)
                loss = torch.zeros(P, device=be.device)
                for t in range(T):
                    x = torch.cat([obs[:, t].expand(P, B, i), state], -1)
                    out = torch.empty(P, B, o + S, device=be.device)
                    be.act_rnn(dims, theta, table, offsets, order, pairs, 0.05, x, out, code)
                    loss += ((out[..., :o] - tgt[:, t]) ** 2).sum((1, 2))
                    state = out[..., o:]
                return -loss / (B * T * o)
            seq_ms = _time(seq, reps)
            steps_ms = _time(steps, max(2, reps // 4))
            rows.append(dict(kind="evaluate", cell=cell, H=H, n=n, P=P, B=B, T=T, seq_ms=round(seq_ms, 3),
                             steps_ms=round(steps_ms, 3), speedup=round(steps_ms / seq_ms, 2)))
            print(json.dumps(rows[-1]), flush=True)
    return rows


class _Hooks(ES):
    def _after_optimize(self, policy):          # any overridden hook selects hooks mode
        super()._after_optimize(policy)


def train_rows(be, gens):
    rows = []
    g = torch.Generator().manual_seed(1)
    obs, tgt = torch.randn(64, 32, 8, generator=g), torch.rand(64, 32, 4, generator=g) * 1.6 - 0.8
    for cls, n_gen in ((ES, gens), (_Hooks, 2)):
        torch.manual_seed(0)
        es = cls(policy_class("gru", True), SequenceAgent, torch.optim.Adam, population_size=256, sigma=0.05,
                 policy_kwargs={"dims": (8, 64, 4)}, agent_kwargs=dict(obs=obs, target=tgt),
                 optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 22, _backend=be)
        es.log = lambda: None
        es.train(n_steps=2)                      # warm-up (and the graph's first sightings in fused mode)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        es.train(n_steps=n_gen)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        rows.append(dict(kind="train", mode="fused" if es._fused else "hooks", P=256, H=64, B=64, T=32,
                         generations=n_gen, gens_per_s=round(n_gen / dt, 3)))
        print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--gens", type=int, default=50)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rnn_sequence_bench needs a CUDA GPU")
    be = CudaBackend()
    q = subprocess.run(["nvidia-smi", "-i", str(be.device.index), "--query-gpu=power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    rows = [dict(kind="device", name=torch.cuda.get_device_name(be.device), power_limit=q.stdout.strip(),
                 library=os.path.basename(_capi.LIB_PATH))]
    print(json.dumps(rows[0]), flush=True)
    rows += kernel_rows(be, a.reps) + train_rows(be, a.gens)
    if a.out:
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
