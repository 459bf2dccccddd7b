#!/usr/bin/env python
"""Population mode measurements (DESIGN.md §9): the per-step act launch (estk_eval_mlp with ESTK_ACTIONS),
the torch alternative a user can write without it, and generations/s of the vectorised CartPole example in
population mode against hooks mode with the same agent.

    python tools/population_rollout_bench.py [--out FILE.json] [--quick]

Per-step act time: CUDA events around many launches after a warm-up.  Achieved bytes/s use the byte count
of ``act_bytes`` (noise row bytes per pair x pairs + theta + observations + outputs) against the 3.35 TB/s
HBM3 figure of the H100 SXM data sheet.  Every step of a generation reads the same noise rows, so at these
sizes they may sit in L2 (50 MB) across steps: the figure is then an L2 rate, not an HBM one.
The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from estorch_b200 import ES  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402

HBM = 3.35e12
NORTH_STAR = [128, 512, 512, 512, 512, 288]


def n_params(dims):
    return sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))


def act_bytes(dims, P, B, noise_bytes):
    n = n_params(dims)
    return noise_bytes * n * (P // 2) + 4 * n + 4 * P * B * (dims[0] + dims[-1])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def time_events(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e-3


def setup(be, dims, P):
    n, pairs = n_params(dims), P // 2
    theta = (torch.rand(n, device=be.device) * 2 - 1) * 0.05
    table = be.alloc(max(1 << 20, (n + 31) // 32 * 32 + 32 * 8192))
    be.fill_noise_table(table, 1)
    t16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, t16) == 0
    offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
    be.make_offsets(2, None, 0, 0, pairs, table.numel(), n, offsets, order)
    return theta, table, t16, offsets, order


def bench_act(be, dims, P, B, iters, warmup):
    theta, table, t16, offsets, order = setup(be, dims, P)
    obs = torch.randn(P, B, dims[0], device=be.device)
    out = be.alloc(P, B, dims[-1])
    res = {"dims": dims, "P": P, "B": B, "n": n_params(dims)}
    for name, tab, tab16, nb in (("table16", None, t16, 2), ("table", table, None, 4)):
        s = time_events(lambda: be.act_mlp(dims, theta, tab, offsets, order, P // 2, 0.02, obs, out, table16=tab16),
                        iters, warmup)
        by = act_bytes(dims, P, B, nb)
        res[name] = {"us_per_step": s * 1e6, "bytes": by, "GBps": by / s / 1e9, "share_of_hbm": by / s / HBM}
    # the torch alternative: rows materialised with estk_perturb_rows, then torch.bmm per layer
    rows = be.alloc(P, n_params(dims))

    def materialise():
        be.perturb_rows(theta, table, offsets, P // 2, 0.02, 0, P, rows)

    def forward():
        h, idx = obs, 0
        for li in range(len(dims) - 1):
            i, o = dims[li], dims[li + 1]
            W = rows[:, idx: idx + i * o].view(P, o, i)
            b = rows[:, idx + i * o: idx + i * o + o]
            idx += i * o + o
            h = torch.baddbmm(b[:, None, :], h, W.transpose(1, 2))
            if li + 2 < len(dims):
                h = torch.relu(h)
        return h
    res["torch_perturb_rows_us"] = time_events(materialise, max(iters // 4, 5), 3) * 1e6
    materialise()
    res["torch_bmm_step_us"] = time_events(forward, iters, warmup) * 1e6
    res["torch_per_step_if_rows_rebuilt_us"] = res["torch_perturb_rows_us"] + res["torch_bmm_step_us"]
    del rows
    torch.cuda.empty_cache()
    return res


def bench_e2e(be, quick):
    import importlib.util
    spec = importlib.util.spec_from_file_location("vector_cartpole", os.path.join(ROOT, "examples", "vector_cartpole.py"))
    vc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(vc)

    class Hooks(ES):
        def _after_optimize(self, policy):      # an overridden hook: the same agent through hooks mode
            super()._after_optimize(policy)
    out = {}
    for name, cls, P, gens in (("population", ES, 1024, 3 if quick else 10), ("hooks", Hooks, 32, 1 if quick else 2)):
        torch.manual_seed(0)
        es = cls(vc.Policy, vc.VectorCartPole, torch.optim.Adam, population_size=P, sigma=0.02,
                 optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 22, _backend=be)
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
    rep = {"card": card(), "act": [bench_act(be, [4, 64, 64, 2], 4096, 1, it, 20),
                                   bench_act(be, [24, 64, 64, 4], 4096, 1, it, 20),
                                   bench_act(be, NORTH_STAR, 1024, 1, max(it // 4, 5), 5)],
           "end_to_end": bench_e2e(be, args.quick)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
