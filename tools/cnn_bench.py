#!/usr/bin/env python
"""Measure the convolutional evaluate (estk_eval_mlp with n_conv in bits 24-31, estk_eval_cnn.cu) on three shapes:
(a) an MNIST-shape classifier, (b) the Atari network without VirtualBatchNorm, (c) a MinAtar-shape network.

For each shape: the evaluate launch time (CUDA events, warmed up, many launches), the achieved fp32 FLOP/s from
the shape's multiply-adds against the H100 SXM data-sheet 67 TFLOP/s, the same evaluate in torch (materialised
rows from estk_perturb_rows, then one grouped ``F.conv2d(groups=members)`` per layer), and generations/s of
``ES.train`` in fused mode and in hooks mode (at a smaller population).  Prints one JSON line per row, the first
with the card and its power limit, and writes them to --out."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from estorch_b200 import ES, DeviceAgent, _capi  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402
from estorch_b200.policy_spec import CNNSpec  # noqa: E402

PEAK_FP32 = 67e12
# name: (input shape, convs, linears, xent, B, populations)
SHAPES = {
    "a_mnist": ((1, 28, 28), [(16, 5, 2, 2), (32, 5, 2, 2)], [10], True, 256, (1024, 4096)),
    "b_atari_no_vbn": ((4, 84, 84), [(16, 8, 4, 0), (32, 4, 2, 0)], [256, 6], False, 32, (1024,)),
    "c_minatar": ((6, 10, 10), [(16, 3, 1, 0)], [128, 4], False, 256, (4096,)),
}


def pack(shape, convs, linears):
    return CNNSpec(tuple(shape), tuple(convs), tuple(linears)).dims


def layer_shapes(shape, convs, linears):
    """[(weight shape, bias length)] of every layer in parameters_to_vector order, and the flattened width."""
    out, (c, h, w) = [], shape
    for o, k, s, p in convs:
        out.append(((o, c, k, k), o))
        c, h, w = o, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    fan = c * h * w
    for o in linears:
        out.append(((o, fan), o))
        fan = o
    return out, c * h * w


def policy_class(shape, convs, linears):
    """An nn.Sequential CNN (ReLU hidden, identity output) of the given shape."""
    class Policy(nn.Module):
        def __init__(self):
            super().__init__()
            mods, c = [], shape[0]
            for o, k, s, p in convs:
                mods += [nn.Conv2d(c, o, k, stride=s, padding=p), nn.ReLU()]
                c = o
            fan = layer_shapes(shape, convs, linears)[1]
            mods.append(nn.Flatten())
            for i, o in enumerate(linears):
                mods.append(nn.Linear(fan, o))
                if i + 1 < len(linears):
                    mods.append(nn.ReLU())
                fan = o
            self.net = nn.Sequential(*mods)

        def forward(self, x):
            return self.net(x)
    return Policy


def macs(shape, convs, linears):
    n, (c, h, w) = 0, shape
    for o, k, s, p in convs:
        h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        n += o * h * w * c * k * k
        c = o
    fan = c * h * w
    for o in linears:
        n += fan * o
        fan = o
    return n


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def torch_eval(be, convs, linears, theta, table, offsets, pairs, obs, tgt, rows, chunk):
    """Materialised rows, then grouped convolutions (members as groups) and batched Linear layers, fp32 (the
    squared error closes it for every shape: the loss is a negligible part of the time)."""
    n_conv = len(convs)
    be.perturb_rows(theta, table, offsets, pairs, 0.05, 0, 2 * pairs, rows)
    shapes, _ = layer_shapes(tuple(obs.shape[1:]), convs, linears)
    rets = []
    for m0 in range(0, 2 * pairs, chunk):
        R = rows[m0: m0 + chunk]
        M, B = R.shape[0], obs.shape[0]
        h = obs.unsqueeze(1).expand(B, M, *obs.shape[1:]).reshape(B, M * obs.shape[1], *obs.shape[2:])
        i = 0
        for li, (ws, bl) in enumerate(shapes):
            sz = ws[0] * (ws[1] if len(ws) == 2 else ws[1] * ws[2] * ws[3])
            w, b = R[:, i: i + sz], R[:, i + sz: i + sz + bl]
            i += sz + bl
            if li < n_conv:
                _, _, s, p = convs[li]
                h = torch.relu(F.conv2d(h, w.reshape(M * ws[0], *ws[1:]), b.reshape(-1), stride=s, padding=p,
                                        groups=M))
                if li == n_conv - 1:
                    h = h.reshape(B, M, -1).transpose(0, 1)
            else:
                h = torch.baddbmm(b[:, None], h, w.reshape(M, *ws).transpose(1, 2))
                if li + 1 < len(shapes):
                    h = torch.relu(h)
        rets.append(-((h - tgt) ** 2).mean((1, 2)))
    return torch.cat(rets)


def kernel_rows(be, reps):
    rows_out = []
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
        for P in pops:
            pairs = P // 2
            offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
            be.make_offsets(3, None, 0, 0, pairs, table.numel(), n, offsets, order)
            ret = be.zeros(P)
            t = _time(lambda: be.eval_cnn(dims, theta, table, offsets, order, pairs, 0.05, obs, tgt, ret[:pairs],
                                          ret[pairs:], act=code), reps)
            flops = 2.0 * macs(shape, convs, linears) * B * P
            row = dict(kind="evaluate", shape=name, B=B, P=P, ms=round(t * 1e3, 3), tflops=round(flops / t / 1e12, 2),
                       of_peak=round(flops / t / PEAK_FP32, 3))
            try:
                rows = be.alloc(P, n)
                c1 = convs[0]
                act1 = c1[0] * ((shape[1] + 2 * c1[3] - c1[1]) // c1[2] + 1) * ((shape[2] + 2 * c1[3] - c1[1]) // c1[2] + 1)
                chunk = max(1, min(P, (1 << 30) // (4 * B * act1)))     # ~1 GB of first-layer activations
                tt = _time(lambda: torch_eval(be, convs, linears, theta, table, offsets, pairs, obs, tgt, rows, chunk),
                           max(2, reps // 5))
                row.update(torch_ms=round(tt * 1e3, 3), speedup=round(tt / t, 2))
                del rows
            except torch.cuda.OutOfMemoryError:
                row.update(torch_ms=None)
            torch.cuda.empty_cache()
            print(json.dumps(row), flush=True)
            rows_out.append(row)
    return rows_out


class _Hooks(ES):
    def _after_optimize(self, policy):          # any overridden hook selects hooks mode
        super()._after_optimize(policy)


def train_rows(be, gens):
    out = []
    for name, (shape, convs, linears, xent, B, pops) in SHAPES.items():
        g = torch.Generator().manual_seed(0)
        obs = torch.rand(B, *shape, generator=g)
        tgt = torch.rand(B, linears[-1], generator=g)
        for cls, P, n_gen in ((ES, pops[0], gens), (_Hooks, 32, 2)):
            torch.manual_seed(0)
            es = cls(policy_class(shape, convs, linears), DeviceAgent, torch.optim.Adam, population_size=P, sigma=0.05,
                     agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy" if xent else "mse"),
                     optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 24, _backend=be)
            es.log = lambda: None
            es.train(n_steps=2)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            es.train(n_steps=n_gen)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            row = dict(kind="train", shape=name, mode="fused" if es._fused else "hooks", P=P, B=B,
                       gens_per_s=round(n_gen / dt, 3))
            print(json.dumps(row), flush=True)
            out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--gens", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    be = CudaBackend()
    q = subprocess.run(["nvidia-smi", "-i", str(be.device.index), "--query-gpu=power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    rows = [dict(kind="device", name=torch.cuda.get_device_name(be.device), power_limit=q.stdout.strip(),
                 library=os.path.basename(_capi.LIB_PATH))]
    print(json.dumps(rows[0]), flush=True)
    rows += kernel_rows(be, a.reps) + train_rows(be, a.gens)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in rows) + "\n")


if __name__ == "__main__":
    main()
