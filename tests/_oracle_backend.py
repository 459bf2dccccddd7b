"""TEST-ONLY stand-in for estorch_b200.backend.CudaBackend built on oracle/.

Lets the host logic (class API, hooks, sharding over gloo, NS bookkeeping) run
on a machine without a GPU.  It is injected through the private ``_backend=``
constructor argument; the product never imports this file or ``oracle``."""
import numpy as np
import torch

from oracle import es_oracle as orc
from estorch_b200.backend import STATE_DTYPE


def _np(t):
    return t.detach().cpu().numpy()


class OracleBackend:
    name = "oracle"

    def __init__(self, tensor_core=False):
        """``tensor_core=True`` also emulates the wgmma evaluate modes ("bf16" / "bf16s",
        with the oracle's bf16 rounding model) so that the host logic around them -- shadows,
        the folded post-update rollout -- runs on CPU."""
        self.device = torch.device("cpu")
        self.sm_count, self.cc, self.launches = 0, (0, 0), 0
        self.tensor_core = tensor_core
        self.centre_folds = 0      # evaluate launches that carried a folded centre task

    def eval_supports_bf16(self, dims, B):
        ok = all(k % 64 == 0 and 64 <= k <= 512 for k in dims[:-1]) and \
            all(n % 32 == 0 and 32 <= n <= 512 for n in dims[1:]) and B % 256 == 0
        return bool(self.tensor_core and ok)

    def eval_supports_f16(self, dims, B):
        return self.eval_supports_bf16(dims, B) and 2 * dims[0] <= 512

    def shadow_f16(self, src, dst, check=True):
        a = _np(src)
        h = a.astype(np.float16)
        dst.copy_(torch.from_numpy(h))
        return int(np.count_nonzero(h.astype(np.float32) != a)) if check else 0

    def shadow_bf16(self, src, dst):
        dst.copy_(torch.from_numpy(orc.round_bf16(_np(src))).to(torch.bfloat16))

    @staticmethod
    def _exact_biases(rows, exact, dims):
        idx = 0
        for i in range(len(dims) - 1):
            idx += dims[i] * dims[i + 1]
            rows[..., idx: idx + dims[i + 1]] = exact[..., idx: idx + dims[i + 1]]
            idx += dims[i + 1]
        return rows

    def alloc(self, *shape, dtype=torch.float32):
        return torch.empty(*shape, dtype=dtype)

    def zeros(self, *shape, dtype=torch.float32):
        return torch.zeros(*shape, dtype=dtype)

    @staticmethod
    def _state(state):
        return state.numpy().view(STATE_DTYPE)

    def fill_noise_table(self, table, seed):
        table.copy_(torch.from_numpy(orc.philox_normal_table(table.numel(), seed)))

    def make_offsets(self, seed, state, gen_host, pair_begin, pairs, table_len, n, offsets_out, order_out=None):
        gen = (int(self._state(state)["generation"][0]) if state is not None else 0) + gen_host
        offs = orc.noise_offsets(seed, gen, pair_begin, pairs, table_len, n)
        offsets_out.copy_(torch.from_numpy(offs))
        if order_out is not None:
            order_out.copy_(torch.from_numpy(np.argsort(offs, kind="stable").astype(np.int32)))

    def perturb_rows(self, theta, table, offsets, pairs, sigma, member_begin, member_count,
                     rows_out=None, eps_out=None):
        pop, eps = orc.sample_population(_np(theta), _np(table), _np(offsets), sigma)
        sl = slice(member_begin, member_begin + member_count)
        if rows_out is not None:
            rows_out.copy_(torch.from_numpy(pop[sl]))
        if eps_out is not None:
            eps_out.copy_(torch.from_numpy(eps[sl]))

    def eval_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                 bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", centre_out=None, **extra):
        pop, _ = orc.sample_population(_np(theta), _np(table), _np(offsets), sigma)
        if precision in ("f16", "bf16", "bf16s"):
            assert self.tensor_core and bc_plus is None
            if precision == "f16":
                t16 = extra["table16"]
                assert t16.dtype == torch.float16 and np.array_equal(_np(t16).astype(np.float32), _np(table))
            rows = pop.copy() if precision != "bf16s" else self._exact_biases(
                orc.sample_population_bf16s(_np(theta), _np(table), _np(offsets), sigma), pop, list(dims))
            fwd = orc.mlp_forward_f16 if precision == "f16" else orc.mlp_forward_bf16
            rets = np.array([orc.synthetic_return(fwd(r, list(dims), _np(obs)), _np(target))
                             for r in rows], dtype=np.float32)
            ret_plus.copy_(torch.from_numpy(rets[:pairs]))
            ret_minus.copy_(torch.from_numpy(rets[pairs:]))
            if centre_out is not None:       # the folded post-update rollout of the previous generation
                self.centre_folds += 1
                self.eval_mlp_center(dims, theta, obs, target, centre_out, precision=precision)
            return
        assert centre_out is None
        rets, bcs = orc.evaluate_population(pop, list(dims), _np(obs), _np(target), bc_obs, bc_dim)
        ret_plus.copy_(torch.from_numpy(rets[:pairs]))
        ret_minus.copy_(torch.from_numpy(rets[pairs:]))
        if bc_plus is not None:
            bc_plus.copy_(torch.from_numpy(bcs[:pairs]))
            bc_minus.copy_(torch.from_numpy(bcs[pairs:]))

    def eval_mlp_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0, precision="fp32", **_):
        th = _np(theta)
        if precision == "f16":
            out = orc.mlp_forward_f16(th, list(dims), _np(obs))
        elif precision in ("bf16", "bf16s"):
            row = th if precision == "bf16" else self._exact_biases(orc.round_bf16(th).copy(), th, list(dims))
            out = orc.mlp_forward_bf16(row, list(dims), _np(obs))
        else:
            out = orc.mlp_forward(th, list(dims), _np(obs))
        ret_out[0] = float(orc.synthetic_return(out, _np(target)))
        if bc_out is not None:
            bc_out.copy_(torch.from_numpy(orc.synthetic_bc(out, bc_obs, bc_dim)))

    def track_best(self, state, reward, theta, best_theta):
        s = self._state(state)
        r = float(reward[0])
        s["episode_reward"] = r
        better = r > float(s["best_reward"][0])
        if better:
            s["best_reward"] = r
            best_theta.copy_(theta)
        s["improved"] = int(better)
        s["generation"] += 1

    @staticmethod
    def _algo(novelty, w_rew, w_nov):
        return "es" if novelty is None else "blend"

    def _raw_sum(self, returns, novelty, w_rew, w_nov, P, table, offsets, pair_begin, pairs_local, n):
        f = np.float32
        c = orc.rank_transformation(_np(returns)).astype(np.float32)
        if novelty is not None:
            c2 = orc.rank_transformation(_np(novelty)).astype(np.float32)
            c = (f(w_rew) * c + f(w_nov) * c2).astype(np.float32)
        tab, offs = _np(table), _np(offsets)
        acc = np.zeros(n, dtype=np.float64)
        for jl in range(pairs_local):
            j = pair_begin + jl
            acc += float(f(c[j] - c[j + P // 2])) * tab[offs[jl]: offs[jl] + n].astype(np.float64)
        return acc.astype(np.float32)

    def _ranks(self, returns, novelty, ranks_out, ranks2_out):
        if ranks_out is not None:
            ranks_out.copy_(torch.from_numpy(orc.compute_ranks(_np(returns)).astype(np.int32)))
        if ranks2_out is not None and novelty is not None:
            ranks2_out.copy_(torch.from_numpy(orc.compute_ranks(_np(novelty)).astype(np.int32)))

    def rank_grad(self, returns, novelty, w_rew, w_nov, P, table, offsets, order, pair_begin, pairs_local,
                  n, grad_sum_out, ranks_out=None, ranks2_out=None, world=1):
        table = table.float()                   # the exact fp16 copy converts back to the fp32 table
        if world > 1:                           # rank-major [world][2][pairs/world] -> member order
            assert table is not None
            pl = P // 2 // world
            unperm = lambda t: None if t is None else t.view(world, 2, pl).permute(1, 0, 2).reshape(-1)
            returns, novelty = unperm(returns), unperm(novelty)
        self._ranks(returns, novelty, ranks_out, ranks2_out)
        grad_sum_out.copy_(torch.from_numpy(self._raw_sum(returns, novelty, w_rew, w_nov, P, table, offsets,
                                                          pair_begin, pairs_local, n)))

    def clamp_adam(self, grad_sum, P, theta, m, v, state, adam, grad_out=None):
        g = (_np(grad_sum) / np.float32(P)).astype(np.float32)
        if theta is None:
            grad_out.copy_(torch.from_numpy(orc.negate_clamp(g)))
            return
        s = self._state(state)
        s["adam_step"] += 1
        th, mm, vv = orc.adam_step(_np(theta), _np(m), _np(v), orc.negate_clamp(g), int(s["adam_step"][0]),
                                   adam.lr, adam.beta1, adam.beta2, adam.eps, adam.weight_decay)
        theta.copy_(torch.from_numpy(th)); m.copy_(torch.from_numpy(mm)); v.copy_(torch.from_numpy(vv))
        if grad_out is not None:
            grad_out.copy_(torch.from_numpy(g))

    def rank_grad_adam(self, returns, novelty, w_rew, w_nov, P, table, offsets, order, theta, m, v, state,
                       adam, ranks_out=None, ranks2_out=None, grad_out=None):
        n = theta.numel()
        tmp = torch.zeros(n)
        returns = returns.reshape(-1)
        self.rank_grad(returns, novelty, w_rew, w_nov, P, table, offsets, order, 0, P // 2, n, tmp,
                       ranks_out, ranks2_out)
        self.clamp_adam(tmp, P, theta, m, v, state, adam, grad_out)

    def knn_novelty(self, bc, archive, k, novelty_out):
        a = _np(archive)
        novelty_out.copy_(torch.tensor([orc.novelty(row, a, k) for row in _np(bc)], dtype=torch.float32))
