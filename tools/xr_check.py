"""Under torchrun: the in-kernel cross-GPU gradient sum (estk_rank_grad_xr_adam) against the same kernel +
NCCL all-reduce + clamp/Adam from identical state: theta', m, v, g compared element by element (bit-identical is
expected at 2 GPUs: a two-term fp32 sum does not depend on its order), repeated to catch races; then timings."""
import os, sys, traceback, torch, torch.distributed as dist
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from estorch_b200.backend import CudaBackend, adam_desc
rank, W = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl")
be = CudaBackend(torch.device("cuda", torch.cuda.current_device()))
P = int(os.environ.get("XR_P", "4096"))
pairs = P // 2
pl = pairs // W
table = be.alloc(1 << 28); be.fill_noise_table(table, 42)
tb16 = be.alloc(table.numel(), dtype=torch.float16); assert be.shadow_f16(table, tb16) == 0


def timed(run, iters=100):
    for _ in range(5):
        run()
    torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record(); torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters * 1e3], device=be.device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


try:
    for n in [int(x) for x in os.environ.get("XR_N", "1001760,6020").split(",")]:
        ad = adam_desc(lr=0.01, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, clamp=1.0)
        offs = be.alloc(pl, dtype=torch.int64); order = be.alloc(pl, dtype=torch.int32)
        be.make_offsets(42, None, 0, rank * pl, pl, table.numel(), n, offs, order)
        mine = be.peer_alloc(be.xr_workspace_bytes(n))
        handles = [None] * W
        dist.all_gather_object(handles, mine[1])
        peers = [mine[0] if r == rank else be.peer_open(handles[r]) for r in range(W)]
        ranks = be.alloc(P, dtype=torch.int32)
        bad = 0
        A = [torch.zeros(n, device=be.device) for _ in range(3)]; sA = be.zeros(32, dtype=torch.uint8); gA = be.alloc(n)
        B = [torch.zeros(n, device=be.device) for _ in range(3)]; sB = be.zeros(32, dtype=torch.uint8); gB = be.alloc(n)
        for it in range(12):
            g = torch.Generator(device="cpu").manual_seed(100 + it)
            ret = torch.randn(P, generator=g).to(be.device)            # same returns on every rank, new every iteration
            be.rank_grad_xr_adam(ret, None, 1.0, 0.0, P, W, rank, tb16, offs, order, rank * pl, pl, peers,
                                 A[0], A[1], A[2], sA, ad, ranks, None, gA)
            be.rank_grad(ret, None, 1.0, 0.0, P, tb16, offs, order, rank * pl, pl, n, gB, ranks, None, world=W)
            dist.all_reduce(gB)
            graw = gB.clone()
            be.clamp_adam(gB, P, B[0], B[1], B[2], sB, ad, None)
            torch.cuda.synchronize()
            gref = graw / P
            neq = [(a != b) for a, b in zip(A, B)] + [gA != gref]
            cnt = [int(x.sum()) for x in neq]
            if any(cnt):
                bad += 1
                idx = torch.nonzero(neq[3] | neq[0]).flatten()
                print(f"rank {rank} n={n} iteration {it}: mismatches theta/m/v/g = {cnt}; first/last index {int(idx[0])}/{int(idx[-1])} "
                      f"of {n}; max |dg|/max|g| = {float((gA - gref).abs().max() / gref.abs().max()):.3e}", flush=True)
        print(f"rank {rank} n={n}: {12 - bad}/12 iterations bit-identical to NCCL all-reduce + clamp/Adam", flush=True)
        ret = torch.randn(P, device=be.device)
        t_xr = timed(lambda: be.rank_grad_xr_adam(ret, None, 1.0, 0.0, P, W, rank, tb16, offs, order, rank * pl, pl, peers,
                                                  A[0], A[1], A[2], sA, ad, ranks, None, gA))
        t_rg = timed(lambda: be.rank_grad(ret, None, 1.0, 0.0, P, tb16, offs, order, rank * pl, pl, n, gB, ranks, None, world=W))

        def nccl_path():
            be.rank_grad(ret, None, 1.0, 0.0, P, tb16, offs, order, rank * pl, pl, n, gB, ranks, None, world=W)
            dist.all_reduce(gB)
            be.clamp_adam(gB, P, B[0], B[1], B[2], sB, ad, None)
        t_nc = timed(nccl_path)
        t_ar = timed(lambda: dist.all_reduce(gB))
        if rank == 0:
            print(f"W={W} n={n}: rank+gradient+NVLink sum+Adam {t_xr:.1f} | rank+partial gradient alone {t_rg:.1f} | "
                  f"rank+partial, NCCL all-reduce, clamp+Adam {t_nc:.1f} | NCCL all-reduce alone {t_ar:.1f}  (us, max over ranks)",
                  flush=True)
except Exception:
    print(f"rank {rank} FAILED:\n" + traceback.format_exc(), flush=True)
dist.destroy_process_group()
