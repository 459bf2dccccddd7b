#!/usr/bin/env python
"""Population mode of a generic convolutional policy (DESIGN.md §4.12, §9): the per-step act launch (estk_act_cnn)
against the torch alternative a user can write without it, hooks mode's per-member forward, and generations/s of
examples/cnn_catch.py in population mode against hooks mode.

    python tools/population_cnn_bench.py [--out FILE.json] [--quick]

Shapes: (a) the example's policy on 1x10x5 grids; (b) the Atari-sized stack 4x84x84, conv 16 k8 s4, conv 32 k4
s2, Linear 256, Linear 6 (§9).  P in {256, 1024, 4096}, B in {1, 4}.  The torch alternative materialises every
member's fp32 row once per generation (estk_perturb_rows) and runs each step as grouped F.conv2d (members as
groups) per conv and torch.baddbmm per Linear.  Times are CUDA events around repeated calls after a warm-up;
the card name, power limit and max SM clock are read in the same run."""
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
from estorch_b200.backend import CudaBackend  # noqa: E402
from estorch_b200.policy_spec import cnn_spec_from_module  # noqa: E402


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


def atari_policy():
    nn = torch.nn
    return nn.Sequential(nn.Conv2d(4, 16, 8, 4), nn.ReLU(), nn.Conv2d(16, 32, 4, 2), nn.ReLU(), nn.Flatten(),
                         nn.Linear(2592, 256), nn.ReLU(), nn.Linear(256, 6))


def torch_step(rows, spec, obs):
    """Materialised rows [M, n], images [M, B, c, h, w] -> [M, B, out]: grouped convolutions, batched Linears."""
    M, B = obs.shape[:2]
    c, h, w = spec.input_shape
    x = obs.transpose(0, 1).reshape(B, M * c, h, w)           # members as groups
    o = 0
    for oc, k, s, p in spec.convs:
        nw = oc * c * k * k
        W, bias = rows[:, o:o + nw].reshape(M * oc, c, k, k), rows[:, o + nw:o + nw + oc].reshape(-1)
        o += nw + oc
        x = torch.relu(F.conv2d(x, W, bias, stride=s, padding=p, groups=M))
        c = oc
    x = x.reshape(B, M, -1).transpose(0, 1)                    # [M, B, C*H*W] in torch's flatten order
    fan = x.shape[-1]
    for i, oc in enumerate(spec.linears):
        W, bias = rows[:, o:o + oc * fan].view(M, oc, fan), rows[:, o + oc * fan:o + oc * fan + oc]
        o += oc * fan + oc
        x = torch.baddbmm(bias[:, None], x, W.transpose(1, 2))
        if i + 1 < len(spec.linears):
            x = torch.relu(x)
        fan = oc
    return x


def kernels(be, name, make_policy, shape, P, B, quick):
    torch.manual_seed(0)
    pol = make_policy().to(be.device)
    spec = cnn_spec_from_module(pol, shape)
    assert spec is not None, name
    theta = torch.nn.utils.parameters_to_vector(pol.parameters()).detach().contiguous()
    n, pairs = theta.numel(), P // 2
    table = be.alloc((n + 31) // 32 * 32 + 32 * 65536)
    be.fill_noise_table(table, 7)
    offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
    be.make_offsets(3, None, 0, 0, pairs, table.numel(), n, offsets, order)
    obs = torch.rand(P, B, *shape, device=be.device)
    out = be.alloc(P, B, spec.out)
    it = 5 if quick else 50
    t_act = time_events(lambda: be.act_cnn(spec.dims, theta, table, offsets, order, pairs, 0.05, obs, out, spec.act),
                        it, 3)
    rows = be.alloc(P, n)
    t_rows = time_events(lambda: be.perturb_rows(theta, table, offsets, pairs, 0.05, 0, P, rows), max(2, it // 5), 1)
    with torch.no_grad():
        ref = torch_step(rows, spec, obs)
        err = float((ref - out).abs().max() / ref.abs().max())
        t_torch = time_events(lambda: torch_step(rows, spec, obs), it, 3)
        x1 = obs[0]                              # hooks mode: one member's forward on its B images
        t_member = time_events(lambda: pol(x1), it, 3)
    return {"shape": name, "P": P, "B": B, "params": n, "act_step_us": t_act * 1e6,
            "torch_rows_once_ms": t_rows * 1e3, "torch_step_us": t_torch * 1e6,
            "act_vs_torch_max_rel_diff": err, "hooks_forward_per_member_step_us": t_member * 1e6,
            "hooks_step_us": t_member * P * 1e6}


def end_to_end(be, ex, P, gens, mode):
    torch.manual_seed(0)
    means, es = ex.train(1, P, backend=be, verbose=False, mode=mode)   # warm-up: workspace growth, first launches
    assert es._population == (mode == "population")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    es.train(n_steps=gens)
    float(es.population_returns.mean())
    dt = (time.perf_counter() - t0) / gens
    return {"mode": mode, "P": P, "episodes_per_member": ex.EPISODES, "generations_per_s": 1 / dt,
            "members_per_s": P / dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    be = CudaBackend()
    ex = load_example("cnn_catch")
    rows = []
    for name, make, shape in (("cnn_catch 1x10x5", ex.policy, (1, 10, 5)), ("atari 4x84x84", atari_policy,
                                                                           (4, 84, 84))):
        for P in (256, 1024, 4096):
            for B in (1, 4):
                rows.append(kernels(be, name, make, shape, P, B, a.quick))
                print(json.dumps(rows[-1]), flush=True)
    e2e = [end_to_end(be, ex, 256, 3, "population"), end_to_end(be, ex, 1024, 3, "population"),
           end_to_end(be, ex, 256, 1, "hooks")]
    rep = {"card": card(), "kernels": rows, "cnn_catch": e2e}
    s = json.dumps(rep, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
