"""Per-role time breakdown of the wgmma evaluate kernel at the north-star shape.

Needs the profile build of the library:
    ESTK_VARIANT=prof ESTK_EXTRA_FLAGS=-DESTK_TC_PROFILE bash estorch_b200/csrc/build.sh
    ESTK_LIBRARY=estorch_b200/lib/libestk_prof.so python tools/eval_profile.py [pairs] [f16|bf16|bf16s]
Every warp sums clock64() deltas per bucket; the table gives, per role, the mean share of a warp's
cycles and the mean cycles per ring stage the warp handled (a producer group forms every fourth stage, a
consumer warpgroup drains every second tile).  "wait other warpgroup" is the tile-order handoff and the
last layer's loss-chain handoff between the two consumer warpgroups.
"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from estorch_b200 import _capi  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402

CONSUMER = ["wait full", "MMA issue .. wait_group", "tile drain + epilogue", "layer: bias + barriers",
            "task: obs load + loss", "wait other warpgroup"]
PRODUCER = ["load issue .. data in registers", "wait empty", "form + store + publish"]


def main():
    pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
    mode = sys.argv[2] if len(sys.argv) > 2 else "f16"
    lib = _capi.load()
    if not hasattr(lib, "estk_tc_profile"):
        sys.exit("eval_profile: ESTK_LIBRARY must name a build made with ESTK_EXTRA_FLAGS=-DESTK_TC_PROFILE")
    be = CudaBackend(torch.device("cuda", 0))
    dims = [128, 512, 512, 512, 512, 288]
    n = sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))
    table = be.alloc(1 << 28); be.fill_noise_table(table, 42)
    offs = be.alloc(pairs, dtype=torch.int64); order = be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
    torch.manual_seed(0)
    theta = torch.randn(n, device=be.device) * 0.05
    obs, tgt = torch.randn(256, 128, device=be.device), torch.randn(256, 288, device=be.device)
    ret = be.zeros(2 * pairs)
    th16 = be.alloc(n, dtype=torch.bfloat16)
    if mode == "f16":
        tb16 = be.alloc(table.numel(), dtype=torch.float16); assert be.shadow_f16(table, tb16) == 0
    else:
        tb16 = be.alloc(table.numel(), dtype=torch.bfloat16); be.shadow_bf16(table, tb16)
    be.shadow_bf16(theta, th16)
    kw = {"table16": tb16} if mode == "f16" else {"theta16": th16, "table16": tb16} if mode == "bf16s" else {}
    run = lambda: be.eval_mlp(dims, theta, table, offs, order, pairs, 0.02, obs, tgt, ret[:pairs], ret[pairs:],
                              precision=mode, **kw)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    warps, cwarps = C.c_int32(), C.c_int32()
    fn = lib.estk_tc_profile
    fn.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    nb = fn(None, C.byref(warps), C.byref(cwarps))
    buf = torch.zeros(sms * warps.value * nb, dtype=torch.int64, device=be.device)
    run(); run()                                     # warm-up, profile off
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn(C.c_void_p(buf.data_ptr()), C.byref(warps), C.byref(cwarps))
    e0.record(); run(); e1.record()
    torch.cuda.synchronize()
    fn(None, C.byref(warps), C.byref(cwarps))
    ms = e0.elapsed_time(e1)
    t = buf.view(sms, warps.value, nb).double().cpu()
    t = t[t.sum(dim=(1, 2)) > 0]                     # CTAs that ran
    stages = 128 * 2 * pairs * 4 // t.shape[0]      # ring stages per CTA: 128 per task, 4 tasks per member
    cons, prod = t[:, :cwarps.value].reshape(-1, nb), t[:, cwarps.value:].reshape(-1, nb)
    print(f"eval {mode} pairs={pairs}: {ms:.3f} ms (profiled launch), {t.shape[0]} CTAs, "
          f"{warps.value} warps/CTA ({cwarps.value} consumer), {stages} stages per CTA")
    for role, rows, names, first, per in (("consumer", cons, CONSUMER, 0, cwarps.value // 4), ("producer", prod, PRODUCER, len(CONSUMER), 4)):
        tot = rows[:, first:first + len(names)].sum(dim=1).mean().item()
        print(f"  {role} warp: {tot / 1e6:.2f} Mcycles")
        for i, name in enumerate(names):
            v = rows[:, first + i].mean().item()
            print(f"    {name:34s} {100 * v / tot:5.1f}%  {v * per / stages:8.0f} cycles/stage")


if __name__ == "__main__":
    main()
