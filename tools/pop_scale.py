"""Population scaling: generations/s and members/s through ES.train as the population grows, and the
rank + gradient call at P in {16384, 32768} of this library against another build (e.g. the parent
commit's, which ranked P > 8192 by an O(P^2) count on global memory), alternated in one process.

    python tools/pop_scale.py [--other-lib path/to/libestk.so] [--out result.json]

Prints one JSON line per measurement, each with the card name and its power limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


class MLP(torch.nn.Module):
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


def es_rate(dims, precision, P, warmup, steps):
    import estorch_b200 as E
    g = torch.Generator().manual_seed(0)
    obs, tgt = torch.randn(256, dims[0], generator=g), torch.randn(256, dims[-1], generator=g)
    torch.manual_seed(0)
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=P, sigma=0.02, policy_kwargs={"dims": dims},
              agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 26,
              log_interval=1 << 30, eval_precision=precision)
    es.log = lambda: None
    es.train(n_steps=warmup)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    es.train(n_steps=steps)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    del es
    torch.cuda.empty_cache()
    return steps / dt


def load_lib(path):
    lib = C.CDLL(path)
    P_ = C.c_void_p
    lib.estk_ctx_create.argtypes = [C.c_int, C.POINTER(P_)]
    lib.estk_rank_grad.argtypes = [P_, P_, P_, C.c_float, C.c_float, C.c_int32, C.c_int32, P_, P_, P_, P_,
                                   C.c_int32, C.c_int32, C.c_int64, P_, P_, P_, P_]
    ctx = P_()
    assert lib.estk_ctx_create(0, C.byref(ctx)) == 0
    return lib, ctx


def rank_grad_compare(libs, P, n=64, reps=50, rounds=5, half=False):
    """estk_rank_grad with each library, alternated; half: the fp16 table form (table16)."""
    rng = np.random.RandomState(P)
    table_len = (n + 31) // 32 * 32 + (1 << 16)
    table = torch.from_numpy(rng.standard_normal(table_len).astype(np.float16).astype(np.float32)).cuda()
    if half:
        table = table.to(torch.float16)
    ret = torch.from_numpy(rng.standard_normal(P).astype(np.float32)).cuda()
    slots = (table_len - (n + 31) // 32 * 32) // 32 + 1
    offs = torch.from_numpy((rng.randint(0, slots, P // 2) * 32).astype(np.int64)).cuda()
    gsum = torch.zeros(n, device="cuda")
    ranks = {k: torch.zeros(P, dtype=torch.int32, device="cuda") for k in libs}
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(name):
        lib, ctx = libs[name]
        tp = C.c_void_p(table.data_ptr())
        rc = lib.estk_rank_grad(ctx, C.c_void_p(ret.data_ptr()), None, 1.0, 0.0, P, 1, None if half else tp,
                                tp if half else None, C.c_void_p(offs.data_ptr()), None, 0, P // 2, n, C.c_void_p(gsum.data_ptr()),
                                C.c_void_p(ranks[name].data_ptr()), None, stream)
        assert rc == 0, rc

    times = {k: [] for k in libs}
    for k in libs:
        for _ in range(3):
            call(k)
    for _ in range(rounds):
        for k in libs:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                call(k)
            b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b) * 1e3 / reps)
    names = list(libs)
    same = all(torch.equal(ranks[names[0]], ranks[k]) for k in names[1:])
    return {k: {"median_us": float(np.median(v)), "min_us": float(np.min(v))} for k, v in times.items()}, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other-lib", default=None, help="another libestk.so to time estk_rank_grad against")
    ap.add_argument("--sizes", default="4096,32768,131072,1048576")
    ap.add_argument("--rank-only", action="store_true", help="only the estk_rank_grad comparison")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pop_scale: needs a CUDA GPU")
    dev = card()
    rows = []

    def emit(r):
        r["gpu"] = dev
        rows.append(r)
        print(json.dumps(r), flush=True)

    if args.other_lib:
        from estorch_b200 import _capi
        libs = {"this": load_lib(_capi.LIB_PATH), "other": load_lib(args.other_lib)}
        for P in (16384, 32768):
            t, same = rank_grad_compare(libs, P)
            emit({"what": "estk_rank_grad", "n": 64, "P": P, "times": t, "ranks_identical": same})
        # the gradient phase at a large n with P > 8192 (fp16 table, the engine's default form)
        t, same = rank_grad_compare(libs, 16384, n=1 << 20, reps=10, half=True)
        emit({"what": "estk_rank_grad", "table": "fp16", "n": 1 << 20, "P": 16384, "times": t, "ranks_identical": same})
    for name, dims, prec in () if args.rank_only else (("cartpole", [4, 64, 64, 2], "fp32"), ("f16_mlp", [64, 256, 256, 32], "f16")):
        for P in (int(s) for s in args.sizes.split(",")):
            steps = max(3, min(200, (1 << 22) // P))
            gps = es_rate(dims, prec, P, warmup=3, steps=steps)
            emit({"what": "ES.train", "policy": name, "dims": dims, "precision": prec, "B": 256, "P": P,
                  "steps": steps, "generations_per_s": gps, "members_per_s": gps * P})
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
