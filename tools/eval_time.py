"""Time the wgmma evaluate kernel alone at the north-star shape (CUDA events, ms per launch)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from estorch_b200.backend import CudaBackend
be = CudaBackend(torch.device("cuda", 0))
dims = [128, 512, 512, 512, 512, 288]
n = sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))
pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
mode = sys.argv[2] if len(sys.argv) > 2 else "f16"
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
for _ in range(3):
    run()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
iters = 20
e0.record()
for _ in range(iters):
    run()
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / iters
print(f"eval {mode} pairs={pairs} ring={os.environ.get('ESTK_TC_RING', 'default')} dbg={os.environ.get('ESTK_TC_DEBUG', '0')}: "
      f"{ms:.4f} ms  {2 * n * 256 * 2 * pairs / ms / 1e9:.1f} TFLOP/s  checksum {float(ret.double().sum()):.9f}")
