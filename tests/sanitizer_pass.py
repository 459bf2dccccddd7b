"""A small pass over the hot kernels for compute-sanitizer (memcheck / racecheck / synccheck): the wgmma evaluate
(default f16 mode, two-tile and one-tile layers, a folded centre task), the fp16-table rank+reduce+Adam and the
multi-GPU form, each checked against the oracle so that a sanitizer run is also a correctness run."""
import os, sys, numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from estorch_b200.backend import CudaBackend, new_state, adam_desc
from oracle import es_oracle as orc
be = CudaBackend(torch.device("cuda", 0))
d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(be.device)
rng = np.random.RandomState(0)
dims, B, pairs = [128, 512, 512, 288], 256, 3
n = orc.mlp_param_count(dims)
table = orc.round_f16(rng.standard_normal((n + 31) // 32 * 32 + 8192).astype(np.float32))
theta = np.concatenate([np.concatenate([rng.uniform(-1, 1, dims[i] * dims[i + 1]) / np.sqrt(dims[i]),
                                        rng.uniform(-1, 1, dims[i + 1]) / np.sqrt(dims[i])]) for i in range(len(dims) - 1)]).astype(np.float32)
obs, tgt = rng.standard_normal((B, dims[0])).astype(np.float32), rng.standard_normal((B, dims[-1])).astype(np.float32)
offs = orc.noise_offsets(5, 0, 0, pairs, table.size, n)
tb, th = d(table), d(theta)
tb16 = be.alloc(table.size, dtype=torch.float16)
assert be.shadow_f16(tb, tb16) == 0
ret, centre = be.zeros(2 * pairs), be.zeros(1)
be.eval_mlp(dims, th, tb, d(offs), None, pairs, 0.02, d(obs), d(tgt), ret[:pairs], ret[pairs:], precision="f16", table16=tb16,
            centre_out=centre)
pop, _ = orc.sample_population(theta, table, offs, 0.02)
want, _ = orc.evaluate_population(pop, dims, obs, tgt)
rel = lambda a, b: float(np.max(np.abs(a - b)) / np.max(np.abs(b)))
assert rel(ret.cpu().numpy(), want) < 3e-5
assert abs(float(centre) - float(orc.synthetic_return(orc.mlp_forward(theta, dims, obs), tgt))) < 3e-5
P = 2 * pairs
m, v, g, ranks = be.zeros(n), be.zeros(n), be.zeros(n), be.zeros(P, dtype=torch.int32)
be.rank_grad_adam(ret, None, 1.0, 0.0, P, tb16, d(offs), None, th, m, v, new_state(be.device), adam_desc(lr=0.01), ranks, None, g)
gw = orc.calculate_grad_pairs(ret.cpu().numpy(), table, offs, n)
assert np.array_equal(ranks.cpu().numpy(), orc.compute_ranks(ret.cpu().numpy())) and rel(g.cpu().numpy(), gw) < 1e-5
part = be.zeros(n)
be.rank_grad(ret, None, 1.0, 0.0, P, tb16, d(offs), None, 0, pairs, n, part, ranks, None, world=1)
assert rel((part / P).cpu().numpy(), gw) < 1e-5
# rank-major returns of a 3-GPU job (pairs_local = 1): [rank][sign][local pair] -- the same ranks, in member order
rm = ret.view(2, pairs).t().contiguous().view(-1)
ranks_rm = be.zeros(P, dtype=torch.int32)
be.rank_grad(rm, None, 1.0, 0.0, P, tb16, d(offs[:1]), None, 0, 1, n, part, ranks_rm, None, world=3)
assert torch.equal(ranks_rm, ranks)
torch.cuda.synchronize()
print("sanitizer_pass ok", rel(ret.cpu().numpy(), want), rel(g.cpu().numpy(), gw))
