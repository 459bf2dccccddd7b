"""Populations beyond 32,768 members: the radix-sort rank phase, the grid-wide pair-order sort and the
per-call growth of the context workspace, through the C ABI and the public ES classes.

Bars: ranks, offsets and order bit-exact; gradients within 1e-5 max-norm relative of the fp64 oracle;
a result computed twice (fp16 vs fp32 table, large vs small launch, graph vs eager) bit-identical.
"""
import numpy as np
import pytest
import torch

from oracle import es_oracle as orc
from conftest import rel_err
from test_api_cpu import MLP as _MLP

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def dev(be, a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(be.device)


def _mix64(z):
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def noise_offsets_np(seed, gen, pair_begin, pairs, table_len, n):
    """orc.noise_offsets, vectorised (uint64 arithmetic wraps like the python ints masked to 64 bits)."""
    nslots = np.uint64(orc.noise_slots(table_len, n))
    base = np.uint64(orc.mix64((seed ^ ((gen * 0xD1342543DE82EF95) & ((1 << 64) - 1))) & ((1 << 64) - 1)))
    with np.errstate(over="ignore"):
        j = base + np.arange(pair_begin, pair_begin + pairs, dtype=np.uint64)
    return (np.uint64(32) * (_mix64(j) % nslots)).astype(np.int64)


def grad_pairs_np(c, table, offsets, n, chunk=2048):
    """orc.calculate_grad_pairs on given centred values c (float32 [P]), in float64, chunked."""
    pairs = len(offsets)
    w = c[:pairs].astype(np.float64) - c[pairs:].astype(np.float64)
    acc = np.zeros(n, dtype=np.float64)
    cols = np.arange(n)
    for s in range(0, pairs, chunk):
        rows = table[offsets[s:s + chunk, None] + cols[None, :]].astype(np.float64)
        acc += w[s:s + chunk] @ rows
    return acc / (2 * pairs)


def test_vectorised_offsets_helper_matches_oracle():
    np.testing.assert_array_equal(noise_offsets_np(0xDEADBEEF12345, 7, 1234, 500, 1 << 22, 4610),
                                  orc.noise_offsets(0xDEADBEEF12345, 7, 1234, 500, 1 << 22, 4610))


def _returns_with_specials(P, seed):
    """Returns with planted ties, +-0, +-inf and NaN (the cases the rank order has rules for)."""
    rng = np.random.RandomState(seed)
    r = rng.standard_normal(P).astype(np.float32)
    r[rng.choice(P, P // 8, replace=False)] = np.round(r[rng.choice(P, P // 8, replace=False)], 1)   # many ties
    k = max(P // 64, 4)
    idx = rng.permutation(P)[:6 * k].reshape(6, k)
    r[idx[0]] = 0.0
    r[idx[1]] = -0.0
    r[idx[2]] = np.inf
    r[idx[3]] = -np.inf
    r[idx[4]] = np.nan
    r[idx[5]] = np.float32(1.5)
    return r


def _rank_major(r, W):
    P = r.size
    pl = P // 2 // W
    return np.ascontiguousarray(r.reshape(2, W, pl).transpose(1, 0, 2).reshape(-1))


@pytest.mark.parametrize("P", [8194, 32768, 32770, 65536, 1 << 20, 1 << 22])
@pytest.mark.parametrize("world", [1, 4])
def test_ranks_bit_exact_against_stable_argsort(be, P, world):
    if (P // 2) % world:
        pytest.skip("world must divide the pairs")
    n, table_len = 64, 1 << 16
    rew = _returns_with_specials(P, P + world)
    nov = _returns_with_specials(P, 3 * P + world)
    table = np.random.RandomState(1).standard_normal(table_len).astype(np.float32)
    offs = noise_offsets_np(5, 0, 0, P // 2, table_len, n)
    ranks = be.zeros(P, dtype=torch.int32)
    ranks2 = be.zeros(P, dtype=torch.int32)
    gsum = be.zeros(n)
    lay = (lambda a: _rank_major(a, world)) if world > 1 else (lambda a: a)
    be.rank_grad(dev(be, lay(rew)), dev(be, lay(nov)), 0.25, 0.75, P, dev(be, table), dev(be, offs), None, 0,
                 P // 2, n, gsum, ranks, ranks2, world=world)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(ranks.cpu().numpy(), orc.compute_ranks(rew))
    np.testing.assert_array_equal(ranks2.cpu().numpy(), orc.compute_ranks(nov))


@pytest.mark.parametrize("P", [65536, 1 << 20])
def test_gradient_and_adam_large_population(be, P):
    from estorch_b200.backend import new_state, write_state, read_state, adam_desc
    n = 4610
    rng = np.random.RandomState(P % 1000)
    table_len = (n + 31) // 32 * 32 + (1 << 20)
    table = np.round(rng.standard_normal(table_len), 2).astype(np.float16).astype(np.float32)   # exact in fp16
    offs = noise_offsets_np(11, 2, 0, P // 2, table_len, n)
    ret = rng.standard_normal(P).astype(np.float32)
    c = orc.center_values(P).astype(np.float32)[orc.compute_ranks(ret)]
    want = grad_pairs_np(c, table, offs, n)
    order = dev(be, np.argsort(offs, kind="stable").astype(np.int32))
    t32, t16 = dev(be, table), dev(be, table).to(torch.float16)
    theta = (rng.standard_normal(n) * 0.1).astype(np.float32)
    out = {}
    for name, t in (("fp32", t32), ("fp16", t16)):
        gsum = be.zeros(n)
        ranks = be.zeros(P, dtype=torch.int32)
        be.rank_grad(dev(be, ret), None, 1.0, 0.0, P, t, dev(be, offs), order, 0, P // 2, n, gsum, ranks)
        st = new_state(be.device)
        write_state(st, adam_step=3)
        th, m, v, g = dev(be, theta), be.zeros(n), be.zeros(n), be.zeros(n)
        be.rank_grad_adam(dev(be, ret), None, 1.0, 0.0, P, t, dev(be, offs), order, th, m, v, st, adam_desc(lr=0.01),
                          None, None, g)
        torch.cuda.synchronize()
        assert read_state(st)["adam_step"] == 4
        np.testing.assert_array_equal(ranks.cpu().numpy(), orc.compute_ranks(ret))
        out[name] = (gsum.cpu().numpy(), g.cpu().numpy(), th.cpu().numpy())
        assert rel_err(out[name][0] / P, want) < 1e-5
        assert rel_err(out[name][1], want) < 1e-5
        th_want, _, _ = orc.adam_step(theta, np.zeros(n, np.float32), np.zeros(n, np.float32),
                                      orc.negate_clamp(out[name][1]), 4)
        assert rel_err(out[name][2], th_want) < 1e-6
    # the fp16 table holds the same values; at this n the two forms split the columns differently, so
    # only the fp32 summation order differs
    for a, b in zip(out["fp32"], out["fp16"]):
        assert rel_err(b, a) < 2e-6


@pytest.mark.parametrize("pairs", [4097, 16384, 16385, 65536, 1 << 19, 1 << 21])
def test_make_offsets_sorted_order_bit_exact(be, pairs):
    from estorch_b200.backend import new_state, write_state
    n, table_len, pair_begin, gen = 4610, 1 << 28, 3 * pairs + 7, 6
    want = noise_offsets_np(0xDEADBEEF12345, gen, pair_begin, pairs, table_len, n)
    want_order = np.lexsort((np.arange(pairs), want)).astype(np.int32)
    st = new_state(be.device)
    write_state(st, generation=gen - 2)                    # device counter + host offset = gen
    offs = be.alloc(pairs, dtype=torch.int64)
    order = be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(0xDEADBEEF12345, st, 2, pair_begin, pairs, table_len, n, offs, order)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(offs.cpu().numpy(), want)
    np.testing.assert_array_equal(order.cpu().numpy(), want_order)
    # a short table: many equal slots, ties broken by the pair index
    offs2 = be.alloc(pairs, dtype=torch.int64)
    be.make_offsets(9, None, 0, 0, pairs, 4096 + 64 * 32, 4096, offs2, order)
    want2 = noise_offsets_np(9, 0, 0, pairs, 4096 + 64 * 32, 4096)
    np.testing.assert_array_equal(offs2.cpu().numpy(), want2)
    np.testing.assert_array_equal(order.cpu().numpy(), np.lexsort((np.arange(pairs), want2)).astype(np.int32))


def _eval_mlp_members(be, dims, precision, theta, table, table16, offs, sigma, obs, tgt, bc_obs, bc_dim, centre):
    pairs = offs.numel()
    rp, rm = be.zeros(pairs), be.zeros(pairs)
    bp, bm = be.zeros(pairs, bc_dim), be.zeros(pairs, bc_dim)
    c = be.zeros(1) if centre else None
    be.eval_mlp(dims, theta, table, offs, None, pairs, sigma, obs, tgt, rp, rm, bp, bm, bc_obs, bc_dim,
                precision=precision, table16=table16, centre_out=c)
    torch.cuda.synchronize()
    return rp.cpu().numpy(), rm.cpu().numpy(), bp.cpu().numpy(), bm.cpu().numpy(), None if c is None else c.item()


@pytest.mark.parametrize("precision", ["fp32", "f16"])
def test_eval_mlp_large_population_matches_small_launches(be, precision):
    """2^16 + 3 pairs in one launch: every member equals the same member evaluated in a launch of the
    size the engine always supported (which the oracle tests cover), bit for bit; a strided sample also
    against the fp32 oracle."""
    dims = [64, 256, 256, 32]
    n = orc.mlp_param_count(dims)
    pairs = (1 << 16) + 3
    rng = np.random.RandomState(3)
    table_len = (n + 31) // 32 * 32 + (1 << 20)
    table = dev(be, rng.standard_normal(table_len).astype(np.float16).astype(np.float32))
    t16 = table.to(torch.float16)
    theta = dev(be, (rng.standard_normal(n) * 0.05).astype(np.float32))
    obs = dev(be, rng.standard_normal((256, 64)).astype(np.float32))
    tgt = dev(be, rng.standard_normal((256, 32)).astype(np.float32))
    offs_np = noise_offsets_np(4, 0, 0, pairs, table_len, n)
    centre = precision == "f16"
    big = _eval_mlp_members(be, dims, precision, theta, table, t16, dev(be, offs_np), 0.02, obs, tgt, 2, 48, centre)
    pick = np.arange(0, pairs, 4099)
    small = _eval_mlp_members(be, dims, precision, theta, table, t16, dev(be, offs_np[pick]), 0.02, obs, tgt, 2, 48,
                              centre)
    for a, b in zip(big[:4], small[:4]):
        np.testing.assert_array_equal(a[pick], b)
    if centre:
        assert big[4] == small[4]
    th, tb = theta.cpu().numpy(), table.cpu().numpy()
    for j in pick[:4]:
        for sgn, ret in ((1.0, big[0]), (-1.0, big[1])):
            row = th + sgn * np.float32(0.02) * tb[offs_np[j]:offs_np[j] + n]
            want = orc.synthetic_return(orc.mlp_forward(row, dims, obs.cpu().numpy()), tgt.cpu().numpy())
            assert abs(ret[j] - want) <= (1e-5 if precision == "fp32" else 2e-3) * abs(want)


@pytest.mark.parametrize("precision", ["fp32", "f16"])
def test_eval_conv_large_population_matches_small_launch(be, precision):
    n_actions, R, B = 6, 2, 2
    pairs = 16385
    layout = orc.atari_param_layout(n_actions)
    n = int(sum(int(np.prod(s)) for _, s in layout)) if isinstance(layout, list) else int(layout[-1])
    rng = np.random.RandomState(5)
    table_len = (n + 31) // 32 * 32 + (1 << 16)
    table = dev(be, rng.standard_normal(table_len).astype(np.float16).astype(np.float32))
    t16 = table.to(torch.float16)
    theta = dev(be, (rng.standard_normal(n) * 0.02).astype(np.float32))
    xref = dev(be, rng.random((R, 4, 84, 84)).astype(np.float32))
    obs = dev(be, rng.random((B, 4, 84, 84)).astype(np.float32))
    tgt = dev(be, rng.standard_normal((B, n_actions)).astype(np.float32))
    offs_np = noise_offsets_np(8, 0, 0, pairs, table_len, n)
    scratch = be.alloc(be.conv_scratch_bytes(R, B, precision), dtype=torch.uint8)

    def run(offs):
        p = offs.size
        rp, rm = be.zeros(p), be.zeros(p)
        be.eval_conv_vbn(n_actions, theta, table, dev(be, offs), None, p, 0.01, xref, obs, tgt, rp, rm, scratch,
                         precision=precision, table16=t16 if precision == "f16" else None)
        torch.cuda.synchronize()
        return rp.cpu().numpy(), rm.cpu().numpy()

    big = run(offs_np)
    pick = np.arange(0, pairs, 1031)
    small = run(offs_np[pick])
    np.testing.assert_array_equal(big[0][pick], small[0])
    np.testing.assert_array_equal(big[1][pick], small[1])
    assert np.all(np.isfinite(big[0])) and np.all(np.isfinite(big[1]))
    # sampled members against the fp32 oracle (eps = sigma * t, then theta +- eps, like the reference), with the
    # bars of the small-population tests: fp32 5e-5 (test_kernels_gpu), f16 1e-5 of the fp32 forward (estk.h)
    th, tb = theta.cpu().numpy(), table.cpu().numpy()
    xr, xo, tg = xref.cpu().numpy(), obs.cpu().numpy(), tgt.cpu().numpy()
    got, want = [], []
    for j in (0, pairs // 2, pairs - 1):
        eps = np.float32(0.01) * tb[offs_np[j]:offs_np[j] + n]
        for row, ret in ((th + eps, big[0][j]), (th - eps, big[1][j])):
            got.append(ret)
            want.append(orc.synthetic_return(orc.atari_forward(row, n_actions, xr, xo), tg))
    assert rel_err(got, want) < (5e-5 if precision == "fp32" else 1e-5)


def test_workspace_grows_per_call_and_refuses_under_capture():
    from estorch_b200.backend import CudaBackend
    be = CudaBackend(torch.device("cuda", 0))       # a fresh context: today's footprint
    n, table_len = 256, 1 << 16
    table = dev(be, np.random.RandomState(0).standard_normal(table_len).astype(np.float32))

    def run(P, seed):
        ret = dev(be, np.random.RandomState(seed).standard_normal(P).astype(np.float32))
        offs = dev(be, noise_offsets_np(1, 0, 0, P // 2, table_len, n))
        g, r = be.zeros(n), be.zeros(P, dtype=torch.int32)
        be.rank_grad(ret, None, 1.0, 0.0, P, table, offs, None, 0, P // 2, n, g, r)
        torch.cuda.synchronize()
        return g.cpu().numpy(), r.cpu().numpy()

    a = run(4096, 1)
    big = run(1 << 20, 2)
    np.testing.assert_array_equal(big[1], orc.compute_ranks(
        np.random.RandomState(2).standard_normal(1 << 20).astype(np.float32)))
    b = run(4096, 1)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])

    fresh = CudaBackend(torch.device("cuda", 0))
    P = 1 << 18
    ret = dev(fresh, np.random.RandomState(3).standard_normal(P).astype(np.float32))
    offs = dev(fresh, noise_offsets_np(1, 0, 0, P // 2, table_len, n))
    g = fresh.zeros(n)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match=r"estk_status -4\).*captured"):
        with torch.cuda.graph(graph):
            fresh.rank_grad(ret, None, 1.0, 0.0, P, table, offs, None, 0, P // 2, n, g)
    torch.cuda.synchronize()
    fresh.rank_grad(ret, None, 1.0, 0.0, P, table, offs, None, 0, P // 2, n, g)   # eagerly it grows and runs
    torch.cuda.synchronize()


def test_es_fused_cartpole_shape_p131072(monkeypatch):
    import estorch_b200 as E
    dims, P, sigma, seed, table_len = [4, 64, 64, 2], 1 << 17, 0.05, 3, 1 << 22
    g = torch.Generator().manual_seed(7)
    obs, tgt = torch.randn(256, 4, generator=g), torch.randn(256, 2, generator=g)
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ESTORCH_B200_GRAPH", mode)
        rec = []

        class R(E.ES):
            def log(self):
                rec.append(dict(returns=self.population_returns.copy(), ranks=self._ranks.cpu().numpy().copy(),
                                grad=self._grad.cpu().numpy().copy()))

        torch.manual_seed(0)
        es = R(_MLP, E.DeviceAgent, torch.optim.Adam, population_size=P, sigma=sigma, policy_kwargs={"dims": dims},
               agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=table_len,
               noise_seed=seed)
        assert es._fused
        theta0 = es._slots[0].theta.cpu().numpy().copy()
        table = es._table.cpu().numpy()
        es.train(n_steps=3)
        torch.cuda.synchronize()
        assert es.population_returns.shape == (P, 1)
        out[mode] = (es._slots[0].theta.cpu().numpy(), rec)
    theta, rec = out["1"]
    np.testing.assert_array_equal(theta, out["0"][0])                     # graph replay == eager
    for x, y in zip(rec, out["0"][1]):
        np.testing.assert_array_equal(x["returns"], y["returns"])
    n = theta0.size
    offs = noise_offsets_np(seed, 0, 0, P // 2, es._table.numel(), n)
    rets = rec[0]["returns"][:, 0]
    np.testing.assert_array_equal(rec[0]["ranks"], orc.compute_ranks(rets))
    c = orc.center_values(P).astype(np.float32)[orc.compute_ranks(rets)]
    assert rel_err(rec[0]["grad"], grad_pairs_np(c, table, offs, n)) < 1e-5


def test_nsra_es_fused_bipedal_shape_p65536():
    import estorch_b200 as E
    dims = [24, 64, 64, 4]
    g = torch.Generator().manual_seed(9)
    obs, tgt = torch.randn(256, 24, generator=g), torch.randn(256, 4, generator=g)
    torch.manual_seed(1)
    np.random.seed(1)
    es = E.NSRA_ES(_MLP, E.DeviceAgent, torch.optim.Adam, population_size=65536, sigma=0.05,
                   policy_kwargs={"dims": dims}, agent_kwargs=dict(obs=obs, target=tgt, bc_obs=64, bc_dim=256),
                   optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 22, meta_population_size=2, k=5)
    es.log = lambda: None
    assert es._fused
    n0 = len(es._archive)
    es.train(n_steps=2)
    torch.cuda.synchronize()
    assert es.population_returns.shape[0] == 65536
    assert len(es._archive) == n0 + 2
    assert all(np.isfinite(s.theta.cpu().numpy()).all() for s in es._slots)


def test_fp16_and_fp32_table_gradients_bit_identical_at_matching_geometry(be):
    """At a large n both table forms take the column-split path (one pass over the pairs per column), so the
    fp32 sums are taken in the same order: the gradients are the same bits."""
    n, P = 1001760, 65536
    rng = np.random.RandomState(21)
    table_len = (n + 31) // 32 * 32 + (1 << 20)
    table = dev(be, rng.standard_normal(table_len).astype(np.float16).astype(np.float32))
    offs = dev(be, noise_offsets_np(13, 0, 0, P // 2, table_len, n))
    ret = dev(be, rng.standard_normal(P).astype(np.float32))
    out = []
    for t in (table, table.to(torch.float16)):
        g = be.zeros(n)
        be.rank_grad(ret, None, 1.0, 0.0, P, t, offs, None, 0, P // 2, n, g)
        torch.cuda.synchronize()
        out.append(g.cpu().numpy())
    np.testing.assert_array_equal(out[0], out[1])


def test_centre_fold_at_the_population_limit(be):
    """The tensor-core evaluate folds the centre rollout into a population launch of 2^21 pairs (P = 2^22):
    same return as the fold in a small launch."""
    dims = [64, 64, 32]
    n = orc.mlp_param_count(dims)
    rng = np.random.RandomState(17)
    table_len = (n + 31) // 32 * 32 + (1 << 18)
    table = dev(be, rng.standard_normal(table_len).astype(np.float16).astype(np.float32))
    t16 = table.to(torch.float16)
    theta = dev(be, (rng.standard_normal(n) * 0.05).astype(np.float32))
    obs = dev(be, rng.standard_normal((256, 64)).astype(np.float32))
    tgt = dev(be, rng.standard_normal((256, 32)).astype(np.float32))
    res = []
    for pairs in (1 << 21, 4):
        offs = dev(be, noise_offsets_np(2, 0, 0, pairs, table_len, n))
        rp, rm, c = be.zeros(pairs), be.zeros(pairs), be.zeros(1)
        be.eval_mlp(dims, theta, table, offs, None, pairs, 0.02, obs, tgt, rp, rm, precision="f16", table16=t16,
                    centre_out=c)
        torch.cuda.synchronize()
        res.append((c.item(), rp[:4].cpu().numpy(), rm[:4].cpu().numpy()))
    assert res[0][0] == res[1][0]
    np.testing.assert_array_equal(res[0][1], res[1][1])
    np.testing.assert_array_equal(res[0][2], res[1][2])


def test_es_f16_deferred_centre_at_the_population_limit():
    """ES with the tensor-core evaluate and log_interval > 1 folds the post-update rollout into the next
    generation's launch: at P = 2^22 that launch runs too."""
    import estorch_b200 as E
    dims = [64, 64, 32]
    g = torch.Generator().manual_seed(5)
    obs, tgt = torch.randn(256, 64, generator=g), torch.randn(256, 32, generator=g)
    torch.manual_seed(0)
    es = E.ES(_MLP, E.DeviceAgent, torch.optim.Adam, population_size=1 << 22, sigma=0.02,
              policy_kwargs={"dims": dims}, agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01},
              noise_table_size=1 << 22, log_interval=3, eval_precision="f16")
    es.log = lambda: None
    assert es._fused and es._precision == "f16"
    es.train(n_steps=3)
    torch.cuda.synchronize()
    assert np.isfinite(es.episode_reward)
    assert es.population_returns.shape == (1 << 22, 1)


def test_hooks_mode_sgd_gradient_equals_fused_gradient_p32770(be):
    """torch.optim.SGD runs the reference's hook control flow (host rollouts); its gradient on a generation's
    returns equals the fused rank + gradient kernel's on the same returns and offsets."""
    import estorch_b200 as E
    dims = [4, 16, 2]
    g = torch.Generator().manual_seed(3)
    obs, tgt = torch.randn(16, 4, generator=g), torch.randn(16, 2, generator=g)
    grads = []

    class H(E.ES):
        def _calculate_grad(self, epsilon):
            out = super()._calculate_grad(epsilon)
            grads.append(torch.as_tensor(out).detach().cpu().numpy().copy())
            return out

    torch.manual_seed(2)
    P = 32770
    es = H(_MLP, E.DeviceAgent, torch.optim.SGD, population_size=P, sigma=0.05, policy_kwargs={"dims": dims},
           agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 16)
    es.log = lambda: None
    assert not es._fused
    es.train(n_steps=1)
    torch.cuda.synchronize()
    rets = es.population_returns[:, 0].astype(np.float32)
    n = es.n_parameters
    offs = noise_offsets_np(es._noise_seed, 0, 0, P // 2, es._table.numel(), n)
    gs = es._be.zeros(n)
    es._be.rank_grad(dev(es._be, rets), None, 1.0, 0.0, P, es._table, dev(es._be, offs), None, 0, P // 2, n, gs)
    torch.cuda.synchronize()
    fused = gs.cpu().numpy() / np.float32(P)
    assert len(grads) == 1 and rel_err(grads[0], fused) < 1e-5
    c = orc.center_values(P).astype(np.float32)[orc.compute_ranks(rets)]
    assert rel_err(fused, grad_pairs_np(c, es._table.cpu().numpy(), offs, n)) < 1e-5


def test_train_n_proc_2_large_population(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import os
    import subprocess
    import sys
    import textwrap
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "user_script.py"
    script.write_text(textwrap.dedent(f"""
        import os, sys, numpy as np, torch
        sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
        import estorch_b200 as E
        from test_api_cpu import MLP
        g = torch.Generator().manual_seed(1)
        obs, tgt = torch.randn(256, 4, generator=g), torch.randn(256, 2, generator=g)
        es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=65536, sigma=0.02,
                  policy_kwargs={{"dims": [4, 64, 64, 2]}}, agent_kwargs=dict(obs=obs, target=tgt),
                  optimizer_kwargs={{"lr": 0.01}}, noise_table_size=1 << 22)
        es.log = lambda: None
        es.train(n_steps=3, n_proc=2)
        torch.cuda.synchronize()
        np.save(os.path.join({str(tmp_path)!r}, f"theta_rank{{es.rank}}.npy"), es._slots[0].theta.cpu().numpy())
    """))
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    np.testing.assert_array_equal(np.load(tmp_path / "theta_rank0.npy"), np.load(tmp_path / "theta_rank1.npy"))
