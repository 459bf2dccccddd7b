"""Timing of the conv + VirtualBatchNorm evaluate at BASELINE config-5 scale (population 1024,
reference batch 128, observation batch B, 4 actions), fp32 CUDA-core kernel vs the "f16"
tensor-core kernel.

    python tools/conv_bench.py [--precision both|fp32|f16] [--B 32] [--launches 20] [--api]

The requested precisions are launched alternately in one process (after one warm-up launch
each); the JSON line reports the median and range of the per-launch times, and algorithmic
TFLOP/s counted from the network's MACs (the f16 kernel's hi/lo split products are not counted,
so both modes are rated on the same work).  --api additionally times generations/s through
ES.train (the tools/config_bench.py config-5 setup) in each mode.  The card name and its power
limit (read-only nvidia-smi query) are part of the record."""
import argparse, json, os, statistics, subprocess, sys, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from estorch_b200.backend import CudaBackend

ap = argparse.ArgumentParser()
ap.add_argument("--precision", default="both", choices=("both", "fp32", "f16"))
ap.add_argument("--B", type=int, default=32)
ap.add_argument("--launches", type=int, default=20)
ap.add_argument("--api", action="store_true")
args = ap.parse_args()
modes = ("fp32", "f16") if args.precision == "both" else (args.precision,)


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


be = CudaBackend(torch.device("cuda", 0))
A, R, B, P = 4, 128, args.B, 1024
n = 677268
pairs = P // 2
table = be.alloc(1 << 26); be.fill_noise_table(table, 42)
tb16 = be.alloc(table.numel(), dtype=torch.float16)
assert be.shadow_f16(table, tb16) == 0
offs = be.alloc(pairs, dtype=torch.int64); order = be.alloc(pairs, dtype=torch.int32)
be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
theta = torch.randn(n, device=be.device) * 0.02
xref, obs, tgt = torch.rand(R, 4, 84, 84, device=be.device), torch.rand(B, 4, 84, 84, device=be.device), torch.randn(B, A, device=be.device)
scratch = {m: torch.empty(be.conv_scratch_bytes(R, B, m), dtype=torch.uint8, device=be.device) for m in modes}
ret = {m: be.zeros(P) for m in modes}


def run(m):
    r = ret[m]
    be.eval_conv_vbn(A, theta, table, offs, order, pairs, 0.02, xref, obs, tgt, r[:pairs], r[pairs:], scratch[m],
                     precision=m, table16=tb16 if m == "f16" else None)


for m in modes:
    run(m)
torch.cuda.synchronize()
times = {m: [] for m in modes}
for _ in range(args.launches):
    for m in modes:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); run(m); b.record(); torch.cuda.synchronize()
        times[m].append(a.elapsed_time(b))
macs = P * ((R + B) * (6400 * 256 + 2592 * 256) + B * (2592 * 256 + 256 * A))
rec = {"card": torch.cuda.get_device_name(0), "power_limit": power_limit(), "P": P, "ref_batch": R, "B": B,
       "n_actions": A, "launches": args.launches, "algorithmic_gflop_per_evaluate": 2 * macs / 1e9, "modes": {}}
for m in modes:
    med = statistics.median(times[m])
    rec["modes"][m] = {"ms_median": med, "ms_min": min(times[m]), "ms_max": max(times[m]),
                       "algorithmic_TFLOPs": 2 * macs / med / 1e9}
if len(modes) == 2:
    d = (ret["f16"] - ret["fp32"]).abs().max() / ret["fp32"].abs().max()
    rec["f16_returns_max_rel_diff_vs_fp32"] = float(d)
    rec["speedup_f16_over_fp32"] = rec["modes"]["fp32"]["ms_median"] / rec["modes"]["f16"]["ms_median"]
print(json.dumps(rec), flush=True)

if args.api:
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import estorch_b200 as E
    from test_api_gpu import AtariPolicy
    g = torch.Generator().manual_seed(0)
    xr = torch.rand(128, 4, 84, 84, generator=g)
    ob, tg = torch.rand(32, 4, 84, 84, generator=g), torch.randn(32, 4, generator=g)

    class Cfg(E.ES):
        def log(self): pass

    api = {}
    for m in modes:
        es = Cfg(AtariPolicy, E.DeviceAgent, torch.optim.Adam, population_size=1024, sigma=0.02,
                 policy_kwargs=dict(n_actions=4, xref=xr), agent_kwargs=dict(obs=ob, target=tg),
                 optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 26, eval_precision=m)
        assert es._fused and es._is_conv and es._precision == m
        es.train(1); torch.cuda.synchronize()
        t0 = time.perf_counter(); es.train(5); torch.cuda.synchronize()
        api[m] = 5 / (time.perf_counter() - t0)
        del es
        torch.cuda.empty_cache()
    print(json.dumps({"card": rec["card"], "power_limit": rec["power_limit"],
                      "config": "conv+VirtualBatchNorm policy pop=1024, xref 128 frames, B=32 (BASELINE config 5), 1 GPU",
                      "generations_per_s": api}), flush=True)
