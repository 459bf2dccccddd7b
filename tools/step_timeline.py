"""Device timeline of one fused generation at N GPUs (run under torchrun; nsys is not in the image).

Eager launches with a CUDA event before and after every phase of `ES._fused_generation` (the evaluate kernel,
the in-place all-gather, the rank + partial-gradient kernel, the all-reduce, clamp + Adam, the small kernels),
averaged over GENS generations: duration of every phase, the gap in front of it (previous phase's end -> this
phase's start, = launch cost not hidden behind the GPU's backlog) and the spread over the ranks.  Then the same
generation replayed from its CUDA graph, for the total."""
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import MLP, synthetic_batch, WORKLOADS
from estorch_b200 import ES, DeviceAgent

GENS = int(os.environ.get("GENS", "70"))
rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
if world > 1:
    dist.init_process_group("nccl")
wl = WORKLOADS[os.environ.get("WORKLOAD", "north_star")]
obs, tgt = synthetic_batch(wl["dims"], wl["batch"])


class Q(ES):
    def log(self):
        pass


def build():
    torch.manual_seed(0)
    return Q(MLP, DeviceAgent, torch.optim.Adam, population_size=wl["population_size"], sigma=wl["sigma"],
             policy_kwargs={"dims": wl["dims"]}, agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01},
             log_interval=10 ** 9)


marks = []


def wrap(owner, name, label):
    f = getattr(owner, name)

    def g(*a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = f(*a, **k)
        e1.record()
        marks.append((label, e0, e1))
        return r
    setattr(owner, name, g)


os.environ["ESTORCH_B200_GRAPH"] = "0"
es = build()
es.train(5)
for name, label in (("make_offsets", "offset hash + sort"), ("eval_mlp", "evaluate (wgmma)"),
                    ("track_best", "best tracking"), ("rank_grad", "rank + partial gradient"),
                    ("rank_grad_adam", "rank + gradient + Adam"), ("clamp_adam", "clamp + Adam"),
                    ("rank_grad_xr_adam", "rank + gradient + NVLink sum + Adam")):
    wrap(es._be, name, label)
wrap(es, "_all_gather_rm", "all-gather returns (in place)")
wrap(es, "_all_reduce", "all-reduce gradient")
es.train(GENS)                                    # ONE call: steady-state generations (post-update rollout folded)
torch.cuda.synchronize()
first = marks[0][0]
starts = [i for i, m in enumerate(marks) if m[0] == first]
gens = [marks[a:b] for a, b in zip(starts[:-1], starts[1:])][5:]
prev_last = [marks[a - 1] for a in starts[:-1]][5:]       # last phase of the previous generation
labels = [m[0] for m in gens[-1]]
gens, prev_last = zip(*[(g, p) for g, p in zip(gens, prev_last) if [m[0] for m in g] == labels])
rows = []
for i, lab in enumerate(labels):
    dur = sum(g[i][1].elapsed_time(g[i][2]) for g in gens) / len(gens)
    gap = sum((p[2] if i == 0 else g[i - 1][2]).elapsed_time(g[i][1]) for g, p in zip(gens, prev_last)) / len(gens)
    rows.append((lab, dur * 1e3, gap * 1e3))
tot = sum(p[2].elapsed_time(g[-1][2]) for g, p in zip(gens, prev_last)) / len(gens) * 1e3
t = torch.tensor([[d, g] for _, d, g in rows] + [[tot, 0.0]], device="cuda")
tmax, tmin = t.clone(), t.clone()
if world > 1:
    dist.all_reduce(tmax, op=dist.ReduceOp.MAX); dist.all_reduce(tmin, op=dist.ReduceOp.MIN)
del es
torch.cuda.empty_cache()

os.environ["ESTORCH_B200_GRAPH"] = "1"
es = build()
es.train(10)
torch.cuda.synchronize()
if world > 1:
    dist.barrier()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); es.train(200); e1.record(); torch.cuda.synchronize()
gr = torch.tensor([e0.elapsed_time(e1) / 200 * 1e3], device="cuda")
if world > 1:
    dist.all_reduce(gr, op=dist.ReduceOp.MAX)
if rank == 0:
    print(f"# one generation of the north-star workload on {world} GPU(s): eager launches, CUDA events around every phase, "
          f"mean of {len(gens)} generations, microseconds (max over ranks [min over ranks])")
    print(f"{'phase':34s} {'duration':>20s} {'gap in front':>20s}")
    for (lab, _, _), mx, mn in zip(rows, tmax.tolist(), tmin.tolist()):
        print(f"{lab:34s} {mx[0]:9.1f} [{mn[0]:8.1f}] {mx[1]:9.1f} [{mn[1]:8.1f}]")
    print(f"{'generation, eager (host-paced)':34s} {tmax[-1][0].item():9.1f} [{tmin[-1][0].item():8.1f}]")
    print(f"{'generation, CUDA-graph replay':34s} {gr.item():9.1f}   (200 generations back to back, max over ranks)")
    print(f"sum of phase durations {sum(x[0] for x in tmax.tolist()[:-1]):.1f} us")
del es
if world > 1:
    dist.destroy_process_group()
