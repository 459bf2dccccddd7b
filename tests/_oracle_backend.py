"""TEST-ONLY stand-in for estorch_b200.backend.CudaBackend built on oracle/.

Lets the host logic (class API, hooks, sharding over gloo, NS bookkeeping) run
on a machine without a GPU.  It is injected through the private ``_backend=``
constructor argument; the product never imports this file or ``oracle``.

``OracleBackend`` serves every evaluate and act entry point the engine calls (all but the
multi-GPU ``peer_*`` ones) with the references of the kind modules: ``_mlp_oracle``,
``_cnn_oracle`` / ``_cnn_tf32_oracle``, ``_rnn_oracle`` / ``_seq_oracle`` and
``_pop_conv_oracle``.  It counts its calls per entry point and records the MLP codes and the
convolutional precisions it saw, so tests can tell which path the engine took."""
import numpy as np
import torch

from oracle import es_oracle as orc
import _cnn_oracle as cnn
import _cnn_tf32_oracle as tf32
import _mlp_oracle as mlp
import _pop_conv_oracle as conv
import _rnn_oracle as rnn
import _seq_oracle as seq
from estorch_b200.backend import STATE_DTYPE
from estorch_b200.batches import batch_indices


def _np(t):
    return t.detach().cpu().numpy()


class OracleBackend:
    name = "oracle"

    def __init__(self, tensor_core=False, tf32=True):
        """``tensor_core=True`` also emulates the wgmma evaluate modes ("f16", "f16_any", "bf16" /
        "bf16s", with the oracle's rounding models) so that the host logic around them -- shadows,
        the folded post-update rollout -- runs on CPU; ``tf32`` is what ``eval_supports_tf32_cnn``
        answers."""
        self.device = torch.device("cpu")
        self.sm_count, self.cc, self.launches = 0, (0, 0), 0
        self.tensor_core, self.tf32 = tensor_core, tf32
        self.centre_folds = 0      # evaluate launches that carried a folded centre task
        self.acts = set()          # every MLP evaluate code seen
        self.cnn_precisions = []   # the precision of every convolutional evaluate
        self.act_calls = self.cnn_calls = self.seq_calls = self.cnn_act_calls = 0
        self.stats_calls = self.conv_act_calls = self.batch_calls = 0

    def eval_supports_bf16(self, dims, B, act=0):
        ok = all(k % 64 == 0 and 64 <= k <= 512 for k in dims[:-1]) and \
            all(n % 32 == 0 and 32 <= n <= 512 for n in dims[1:]) and B % 256 == 0
        return bool(self.tensor_core and ok and act in mlp.CODES)

    def eval_supports_f16(self, dims, B, act=0):
        return self.eval_supports_bf16(dims, B, act) and 2 * dims[0] <= 512

    def eval_supports_f16_any(self, dims, B, act=0):
        return self.tensor_core and B >= 1 and act in mlp.CODES

    def eval_supports_tf32_cnn(self, dims, B, act=0):
        return self.tf32

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

    def _rows(self, theta, table, offsets, sigma, dims=None, precision="fp32", table16=None):
        """Each member's parameters [M, n]: theta as one row for a centre call (``offsets`` None), else
        ``sample_population``'s [theta + eps; theta - eps].  ``table16`` is the exact fp16 copy of
        ``table``.  "bf16s" rows are rounded as that kernel forms them, the biases exact."""
        th = _np(theta)
        if offsets is None:
            rows = th[None, :]
            if precision == "bf16s":
                rows = self._exact_biases(orc.round_bf16(rows).copy(), rows, list(dims))
            return rows
        if table16 is not None:
            assert table16.dtype == torch.float16
            if table is not None:
                assert np.array_equal(_np(table16).astype(np.float32), _np(table))
            table = table16.float()
        rows, _ = orc.sample_population(th, _np(table), _np(offsets), sigma)
        if precision == "bf16s":
            rows = self._exact_biases(orc.sample_population_bf16s(th, _np(table), _np(offsets), sigma), rows,
                                      list(dims))
        return rows

    @staticmethod
    def _write(rets, bcs, pairs, ret_plus, ret_minus, bc_plus, bc_minus):
        """Returns [M] and bcs [M, bc_dim] into the outputs: the centre's in ``ret_plus[0]`` / ``bc_plus``
        when ``ret_minus`` is None, else the + members first, then their mirrors."""
        if ret_minus is None:
            ret_plus[0] = float(rets[0])
            if bc_plus is not None:
                bc_plus.copy_(torch.from_numpy(np.ascontiguousarray(bcs[0])))
            return
        ret_plus.copy_(torch.from_numpy(rets[:pairs]))
        ret_minus.copy_(torch.from_numpy(rets[pairs:]))
        if bc_plus is not None:
            bc_plus.copy_(torch.from_numpy(np.ascontiguousarray(bcs[:pairs])))
            bc_minus.copy_(torch.from_numpy(np.ascontiguousarray(bcs[pairs:])))

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

    def sample_batch(self, seed, state, gen_host, obs_src, obs_dst, tgt_src, tgt_dst, index_out=None):
        g = gen_host + (int(self._state(state)["generation"][0]) if state is not None else 0)
        idx = torch.from_numpy(batch_indices(seed, g, obs_src.shape[0], obs_dst.shape[0]))
        obs_dst.copy_(obs_src[idx])
        tgt_dst.copy_(tgt_src[idx])
        if index_out is not None:
            index_out.copy_(idx)
        self.batch_calls += 1
        self.launches += 1

    # ---------------------------------------------------------------- MLP evaluate and act modes
    def eval_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                 bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", centre_out=None, act=0, **extra):
        self.acts.add(act)
        assert act in mlp.CODES, hex(act)
        if precision != "fp32":
            assert self.tensor_core and bc_plus is None
        assert centre_out is None or precision not in ("fp32", "f16_any")
        t16 = extra["table16"] if precision in ("f16", "f16_any") else None
        rows = self._rows(theta, table, offsets, sigma, dims, precision, t16)
        rets, bcs = mlp.evaluate_population(rows, dims, _np(obs), _np(target), act, precision, bc_obs, bc_dim)
        self._write(rets, bcs, pairs, ret_plus, ret_minus, bc_plus, bc_minus)
        if centre_out is not None:       # the folded post-update rollout of the previous generation
            self.centre_folds += 1
            self.eval_mlp_center(dims, theta, obs, target, centre_out, precision=precision, act=act)

    def eval_mlp_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0, precision="fp32",
                        act=0, **_):
        self.acts.add(act)
        rows = self._rows(theta, None, None, 0.0, dims, precision)
        rets, bcs = mlp.evaluate_population(rows, dims, _np(obs), _np(target), act, precision, bc_obs, bc_dim)
        self._write(rets, bcs, 1, ret_out, None, bc_out, None)

    def act_mlp(self, dims, theta, table, offsets, order, pairs, sigma, obs, out, act=0, table16=None):
        self.act_calls += 1
        dims = [int(d) for d in dims]
        rows = self._rows(theta, table, offsets, sigma, table16=table16)
        assert tuple(obs.shape) == (rows.shape[0], obs.shape[1], dims[0]) == tuple(out.shape[:2]) + (dims[0],)
        out.copy_(torch.from_numpy(mlp.act_forward(rows, dims, _np(obs), (act & 0xffff) | mlp.ACTIONS)))

    # ---------------------------------------------------------------- recurrent step and sequence evaluate
    def act_rnn(self, dims, theta, table, offsets, order, pairs, sigma, obs, out, act, table16=None):
        self.act_calls += 1
        dims = [int(d) for d in dims]
        cell = rnn.cell_of(act)
        rows = self._rows(theta, table, offsets, sigma, table16=table16)
        S = rnn.state_width(cell, dims[1])
        assert tuple(obs.shape) == (rows.shape[0], obs.shape[1], dims[0] + S)
        assert tuple(out.shape) == (rows.shape[0], obs.shape[1], dims[2] + S)
        out.copy_(torch.from_numpy(rnn.step32(rows, cell, dims, _np(obs), bool(act & mlp.ACT_OUT_TANH))))

    def eval_rnn_seq(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                     bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", act=0):
        assert precision == "fp32"
        self.seq_calls += 1
        dims = [int(d) for d in dims]
        rows = self._rows(theta, table, offsets, sigma)
        B, T = obs.shape[:2]
        assert tuple(obs.shape) == (B, T, dims[0]) and tuple(target.shape) == (B, T, dims[2])
        y = seq.seq_outputs32(rows, rnn.cell_of(act), dims, _np(obs), bool(act & mlp.ACT_OUT_TANH))
        rets = seq.seq_returns32(y, _np(target), bool(act & mlp.LOSS_XENT))
        bcs = y[:, :bc_obs].reshape(len(rows), -1)[:, :bc_dim]
        self._write(rets, bcs, pairs, ret_plus, ret_minus, bc_plus, bc_minus)

    def eval_rnn_seq_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0,
                            precision="fp32", act=0):
        self.eval_rnn_seq(dims, theta, None, None, None, 1, 0.0, obs, target, ret_out, None, bc_out, None, bc_obs,
                          bc_dim, precision=precision, act=act)

    # ---------------------------------------------------------------- convolutional evaluate and act modes
    def eval_cnn(self, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                 bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", act=0):
        self.cnn_precisions.append(precision)
        assert precision in ("fp32", "tf32") and (act >> 24) & 0xff
        self.cnn_calls += 1
        rows = self._rows(theta, table, offsets, sigma)
        if precision == "tf32":
            y = np.stack([tf32.forward_tf32(r, dims, act, _np(obs)) for r in rows])
            rets = tf32.returns64(y, _np(target), act).astype(np.float32)
            bcs = y[:, :bc_obs].reshape(len(rows), -1)[:, :bc_dim].astype(np.float32)
        else:
            y = np.stack([cnn.forward(r, dims, act, _np(obs)) for r in rows])
            rets = cnn.returns_of(y, _np(target), bool(act & mlp.LOSS_XENT))
            bcs = y[:, :bc_obs].reshape(len(rows), -1)[:, :bc_dim]
        self._write(rets, bcs, pairs, ret_plus, ret_minus, bc_plus, bc_minus)

    def eval_cnn_center(self, dims, theta, obs, target, ret_out, bc_out=None, bc_obs=0, bc_dim=0,
                        precision="fp32", act=0):
        self.eval_cnn(dims, theta, None, None, None, 1, 0.0, obs, target, ret_out, None, bc_out, None, bc_obs,
                      bc_dim, precision=precision, act=act)

    def act_cnn(self, dims, theta, table, offsets, order, pairs, sigma, obs, out, act):
        self.cnn_act_calls += 1
        assert (int(act) >> 24) & 0xff and not int(act) & (0xff << 16)
        rows = self._rows(theta, table, offsets, sigma)
        x = _np(obs)
        assert x.ndim == 5 and x.shape[0] == rows.shape[0] and tuple(out.shape) == (rows.shape[0], x.shape[1],
                                                                                    int(dims[-1]))
        out.copy_(torch.from_numpy(np.stack([cnn.forward(r, dims, act, xm) for r, xm in zip(rows, x)])))

    def act_conv_vbn(self, n_actions, theta, table, offsets, order, pairs, sigma, xref, obs, out, stats,
                     table16=None):
        rows = self._rows(theta, table, offsets, sigma, table16=table16)
        assert tuple(stats.shape) == (rows.shape[0], conv.STATS_FLOATS)
        if xref is not None:
            self.stats_calls += 1
            stats.copy_(torch.from_numpy(conv.conv_stats(rows, int(n_actions), _np(xref))))
        if obs is not None:
            self.conv_act_calls += 1
            assert tuple(obs.shape) == (rows.shape[0], obs.shape[1], 4, 84, 84)
            assert tuple(out.shape) == (rows.shape[0], obs.shape[1], int(n_actions))
            out.copy_(torch.from_numpy(conv.conv_act(rows, int(n_actions), _np(stats), _np(obs))))

    # ---------------------------------------------------------------- generation bookkeeping and update
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
