#!/usr/bin/env python
"""Recurrent population mode measurements (DESIGN.md §9): the per-step act launch of a GRUCell / LSTMCell +
Linear head policy (estk_eval_mlp with ESTK_CELL_GRU / ESTK_CELL_LSTM and ESTK_ACTIONS) from the fp16 and
the fp32 noise table, against the torch alternative a user can write without it (rows materialised once per
generation with estk_perturb_rows, then batched matmuls per step), and generations/s of the recall task.

    python tools/population_rnn_bench.py [--out FILE.json] [--quick]

P = 4096, B = 1, in 24, out 4, H in {64, 128, 256}.  Per-step act time: CUDA events around many launches after
a warm-up.  Achieved bytes/s use the noise-row bytes per pair x pairs + theta + observations, state and
outputs, against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet; every step of a generation reads the
same noise rows, so where they fit in L2 (50 MB) the figure is an L2 rate.  The card name and power limit are
read in the same run."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from estorch_b200 import ES  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402
from population_rollout_bench import HBM, card, time_events  # noqa: E402

CELL_CODE = {"gru": 8, "lstm": 9}


def n_params(cell, dims):
    i, h, o = dims
    return (3 if cell == "gru" else 4) * h * (i + h + 2) + o * (h + 1)


def bench_act(be, cell, dims, P, B, iters, warmup):
    n, pairs = n_params(cell, dims), P // 2
    i, H, o = dims
    S = H if cell == "gru" else 2 * H
    theta = (torch.rand(n, device=be.device) * 2 - 1) / H ** 0.5
    table = be.alloc(max(1 << 20, (n + 31) // 32 * 32 + 32 * 8192))
    be.fill_noise_table(table, 1)
    t16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, t16) == 0
    offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
    be.make_offsets(2, None, 0, 0, pairs, table.numel(), n, offsets, order)
    xs = torch.randn(P, B, i + S, device=be.device)
    out = be.alloc(P, B, o + S)
    res = {"cell": cell, "dims": list(dims), "P": P, "B": B, "n": n}
    for name, tab, tab16, nb in (("table16", None, t16, 2), ("table", table, None, 4)):
        s = time_events(lambda: be.act_rnn(dims, theta, tab, offsets, order, pairs, 0.02, xs, out, CELL_CODE[cell],
                                           table16=tab16), iters, warmup)
        by = nb * n * pairs + 4 * n + 4 * P * B * (i + o + 2 * S)
        res[name] = {"us_per_step": s * 1e6, "bytes": by, "GBps": by / s / 1e9, "share_of_hbm": by / s / HBM}
    # the torch alternative: rows once per generation, then per step the gates as two baddbmm, the cell update,
    # and the head as one more baddbmm
    rows = be.alloc(P, n)
    G = 3 if cell == "gru" else 4
    GH = G * H
    w_ih = rows[:, :GH * i].view(P, GH, i)
    w_hh = rows[:, GH * i:GH * (i + H)].view(P, GH, H)
    b_ih = rows[:, GH * (i + H):GH * (i + H + 1)]
    b_hh = rows[:, GH * (i + H + 1):GH * (i + H + 2)]
    w_o = rows[:, GH * (i + H + 2):GH * (i + H + 2) + o * H].view(P, o, H)
    b_o = rows[:, GH * (i + H + 2) + o * H:]
    x, h, c = xs[..., :i], xs[..., i:i + H], xs[..., i + H:]

    def materialise():
        be.perturb_rows(theta, table, offsets, pairs, 0.02, 0, P, rows)

    def step():
        a = torch.baddbmm(b_ih[:, None, :], x, w_ih.transpose(1, 2))
        b = torch.baddbmm(b_hh[:, None, :], h, w_hh.transpose(1, 2))
        if cell == "gru":
            ar, az, an = a.chunk(3, -1)
            br, bz, bn = b.chunk(3, -1)
            r, z = torch.sigmoid(ar + br), torch.sigmoid(az + bz)
            nn_ = torch.tanh(an + r * bn)
            hn = torch.lerp(nn_, h, z)
        else:
            gi, gf, gg, go = (a + b).chunk(4, -1)
            cn = torch.sigmoid(gf) * c + torch.sigmoid(gi) * torch.tanh(gg)
            hn = torch.sigmoid(go) * torch.tanh(cn)
        return torch.baddbmm(b_o[:, None, :], hn, w_o.transpose(1, 2)), hn
    res["torch_perturb_rows_us"] = time_events(materialise, max(iters // 4, 5), 3) * 1e6
    materialise()
    res["torch_step_us"] = time_events(step, iters, warmup) * 1e6
    res["torch_per_step_if_rows_rebuilt_us"] = res["torch_perturb_rows_us"] + res["torch_step_us"]
    del rows
    torch.cuda.empty_cache()
    return res


def bench_e2e(be, quick):
    from _rnn_oracle import RecallAgent, policy_class

    class Hooks(ES):
        def _after_optimize(self, policy):      # an overridden hook: the same agent through hooks mode
            super()._after_optimize(policy)
    out = {}
    for name, cls, P, gens in (("population", ES, 1024, 3 if quick else 10), ("hooks", Hooks, 16, 1 if quick else 2)):
        torch.manual_seed(0)
        es = cls(policy_class("gru", True), RecallAgent, torch.optim.Adam, population_size=P, sigma=0.05,
                 policy_kwargs={"dims": (4, 32, 3)}, optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 20,
                 _backend=be)
        es.log = lambda: None
        assert es._population == (name == "population")
        es.train(n_steps=1)                      # warm-up generation
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        es.train(n_steps=gens)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        out[name] = {"P": P, "generations": gens, "seconds": dt, "generations_per_s": gens / dt,
                     "member_episodes_per_s": gens * P / dt}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON report to this file")
    ap.add_argument("--quick", action="store_true", help="fewer iterations (a rehearsal, not a measurement)")
    args = ap.parse_args()
    be = CudaBackend()
    it = 20 if args.quick else 200
    rep = {"card": card(),
           "act": [bench_act(be, cell, (24, H, 4), 4096, 1, it, 20) for cell in ("gru", "lstm") for H in (64, 128, 256)],
           "end_to_end": bench_e2e(be, args.quick)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
