#!/usr/bin/env python
"""Population mode of the conv + VirtualBatchNorm policy (DESIGN.md §4.7, §9): the stats launch, the per-step
act launch (estk_eval_conv_vbn with n_actions | ESTK_ACTIONS) from table16 and from table, the torch
alternative a user can write without it, hooks mode's per-member forward, and generations/s of the
pixel-Catch example in population mode against hooks mode.

    python tools/population_conv_bench.py [--out FILE.json] [--quick]

Times are CUDA events around repeated launches after a warm-up.  The act step's floor is fc1's noise alone:
pairs x 663,552 values x 2 bytes (table16) at the 3.35 TB/s HBM3 figure of the H100 SXM data sheet.  The
card name and power limit are read in the same run."""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from estorch_b200 import ES, _capi  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402

HBM = 3.35e12
A, R = 4, 128
FC1_W = 256 * 2592


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


def load_example(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "examples", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def setup(be, pc, P):
    torch.manual_seed(0)
    xref = torch.rand(R, 4, 84, 84, device=be.device)
    pol = pc.Policy(A, xref)
    theta = torch.nn.utils.parameters_to_vector(pol.parameters()).detach().to(be.device).contiguous()
    n, pairs = theta.numel(), P // 2
    table = be.alloc((n + 31) // 32 * 32 + 32 * 65536)
    be.fill_noise_table(table, 7)
    t16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, t16) == 0
    offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
    be.make_offsets(3, None, 0, 0, pairs, table.numel(), n, offsets, order)
    obs = torch.rand(P, 1, 4, 84, 84, device=be.device)
    return pol.to(be.device), theta, table, t16, offsets, order, xref, obs


def torch_step(rows, stats, obs, P):
    """Materialised rows + precomputed stats: grouped convolutions and batched fc layers, one step."""
    o = 0
    sz = [16 * 4 * 64, 16, 16, 16, 32 * 16 * 16, 32, 32, 32, FC1_W, 256, A * 256, A]
    parts = []
    for s in sz:
        parts.append(rows[:, o:o + s])
        o += s
    w1, b1, _, _, w2, b2, _, _, f1w, f1b, f2w, f2b = parts
    a1, c1 = stats[:, :6400].view(P, 16, 20, 20), stats[:, 6400:12800].view(P, 16, 20, 20)
    a2, c2 = stats[:, 12800:15392].view(P, 32, 9, 9), stats[:, 15392:].view(P, 32, 9, 9)
    x = F.conv2d(obs.view(1, P * 4, 84, 84), w1.reshape(P * 16, 4, 8, 8), b1.reshape(-1), stride=4, groups=P)
    x = torch.relu(x.view(P, 16, 20, 20) * a1 + c1)
    x = F.conv2d(x.view(1, P * 16, 20, 20), w2.reshape(P * 32, 16, 4, 4), b2.reshape(-1), stride=2, groups=P)
    x = torch.relu(x.view(P, 32, 9, 9) * a2 + c2).view(P, 1, 2592)
    h = torch.relu(torch.bmm(x, f1w.view(P, 256, 2592).transpose(1, 2)) + f1b[:, None])
    return torch.bmm(h, f2w.view(P, A, 256).transpose(1, 2)) + f2b[:, None]


def kernels(be, pc, P, quick):
    pol, theta, table, t16, offsets, order, xref, obs = setup(be, pc, P)
    pairs = P // 2
    stats = be.alloc(P, _capi.ESTK_CONV_VBN_STATS_FLOATS)
    out = be.alloc(P, 1, A)
    it = 3 if quick else 10
    t_stats = time_events(lambda: be.act_conv_vbn(A, theta, table, offsets, order, pairs, 0.02, xref, None, None,
                                                  stats), it, 1)
    t_act16 = time_events(lambda: be.act_conv_vbn(A, theta, None, offsets, order, pairs, 0.02, None, obs, out, stats,
                                                  table16=t16), 10 * it, 3)
    t_act32 = time_events(lambda: be.act_conv_vbn(A, theta, table, offsets, order, pairs, 0.02, None, obs, out,
                                                  stats), 10 * it, 3)
    rows = be.alloc(P, theta.numel())
    t_rows = time_events(lambda: be.perturb_rows(theta, table, offsets, pairs, 0.02, 0, P, rows), it, 1)
    with torch.no_grad():
        t_torch = time_events(lambda: torch_step(rows, stats, obs.view(P, 4, 84, 84), P), 10 * it, 3)
        # hooks mode: the reference forward of one member on one frame (the xref pass included), P of them
        x1 = obs[0]
        t_member = time_events(lambda: pol(x1), 10 * it, 3)
    floor = pairs * FC1_W * 2 / HBM
    return {"P": P, "B": 1, "A": A, "R": R,
            "stats_launch_ms": t_stats * 1e3,
            "act_step_table16_us": t_act16 * 1e6, "act_step_table_us": t_act32 * 1e6,
            "act_fc1_noise_floor_us": floor * 1e6, "act_step_fraction_of_floor": floor / t_act16,
            "torch_rows_once_ms": t_rows * 1e3, "torch_step_us": t_torch * 1e6,
            "hooks_forward_per_member_step_us": t_member * 1e6, "hooks_step_us": t_member * P * 1e6}


class _HooksES(ES):
    def _after_optimize(self, policy):          # any overridden hook selects hooks mode
        super()._after_optimize(policy)


def end_to_end(be, pc, P, gens, hooks=False):
    torch.manual_seed(0)
    xref = pc.reference_batch()
    cls = _HooksES if hooks else ES
    es = cls(pc.Policy, pc.Catch, torch.optim.Adam, population_size=P, sigma=0.02,
             policy_kwargs={"n_actions": 3, "xref": xref.to(be.device)}, optimizer_kwargs={"lr": 0.01},
             noise_table_size=1 << 24, device=be.device, _backend=be)
    assert es._population != hooks
    es.log = lambda: None
    es.train(n_steps=1)                          # warm-up: workspace growth, first launches
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    es.train(n_steps=gens)
    float(es.population_returns.mean())
    dt = (time.perf_counter() - t0) / gens
    return {"mode": "hooks" if hooks else "population", "P": P, "episodes_per_member": pc.EPISODES,
            "generations_per_s": 1 / dt, "member_episodes_per_s": P * pc.EPISODES / dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    be = CudaBackend()
    pc = load_example("pixel_catch")
    rep = {"card": card(), "kernels": [kernels(be, pc, P, a.quick) for P in (100, 1024)],
           "pixel_catch": [end_to_end(be, pc, 100, 3), end_to_end(be, pc, 1024, 3),
                           end_to_end(be, pc, 8, 1, hooks=True)]}
    s = json.dumps(rep, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
