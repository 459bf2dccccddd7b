"""The 16-bit tensor-core MLP evaluate (eval_mlp_tc_kernel, and eval_mlp_tc_stream_kernel behind "f16_any") against
its float64 restatement (tests/_tc_mlp_model.py), output by output.

Every output of every member is read back through the behaviour characteristics (bc_obs = B, bc_dim = B * out), so an
error confined to one tile, one ring stage or one task of the persistent loop shows in the outputs it touched:
    - the roundings, bit for bit through the public entry: one-hot observations give y = fl32(W16 + b) (the weight
      formation of both signs), identity weights the x_hi + x_lo split, two identity layers rn16(act(y));
    - every output of every member and of the centre within its bound, on shapes whose task groups outnumber the
      resident clusters at least twice, and against the float64 forward of the exact fp32 rows at a looser bar;
    - every return against the kernel's own outputs, within the bound of its fp32 reduction (the loss chain apart
      from the GEMM);
    - a NaN observation row gives NaN in that row only, and an infinite observation gives the non-finite outputs it
      gives in fp32."""
import numpy as np
import pytest
import torch

import _mlp_oracle as mlp
import _tc_mlp_model as tcm
from oracle import es_oracle as orc

pytestmark = pytest.mark.gpu

CODES = mlp.CODES


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def dev(be, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(be.device)


def targets(rng, B, N, code):
    loss = mlp.decode(code)[2]
    if loss == "accuracy":
        return np.eye(N, dtype=np.float32)[rng.randint(0, N, B)]
    if loss == "xent":
        t = rng.uniform(0, 1, (B, N)) ** 4
        return (t / t.sum(1, keepdims=True)).astype(np.float32)
    return rng.standard_normal((B, N)).astype(np.float32)


def problem(dims, B, pairs, code=0, seed=5, w_scale=1.0, obs_scale=1.0):
    rng = np.random.RandomState(seed)
    n = orc.mlp_param_count(dims)
    table_len = (n + 31) // 32 * 32 + (1 << 14)
    table = orc.round_f16(rng.standard_normal(table_len).astype(np.float32))
    theta = np.concatenate([np.concatenate([rng.uniform(-1, 1, k * m), rng.uniform(-1, 1, m)]) * w_scale / np.sqrt(k)
                            for k, m in zip(dims[:-1], dims[1:])]).astype(np.float32)
    obs = (rng.standard_normal((B, dims[0])) * obs_scale).astype(np.float32)
    offs = orc.noise_offsets(11, 0, 0, pairs, table_len, n)
    return theta, table, obs, targets(rng, B, dims[-1], code), offs


class Run:
    """One population launch of ``mode`` with every output read back, and the centre evaluation with its outputs."""

    def __init__(self, be, mode, dims, code, theta, table, obs, tgt, offs, sigma, centre_out=False):
        P, B, N = len(offs), obs.shape[0], dims[-1]
        self.th, tb, self.ob, self.tg = dev(be, theta), dev(be, table), dev(be, obs), dev(be, tgt)
        self.kw, self.ckw = {}, {}
        if tcm.kind(mode) == "f16":
            tb16 = be.alloc(table.size, dtype=torch.float16)
            assert be.shadow_f16(tb, tb16) == 0
            self.kw = {"table16": tb16}
        elif mode == "bf16s":
            th16, tb16 = be.alloc(theta.size, dtype=torch.bfloat16), be.alloc(table.size, dtype=torch.bfloat16)
            be.shadow_bf16(self.th, th16)
            be.shadow_bf16(tb, tb16)
            self.kw, self.ckw = {"theta16": th16, "table16": tb16}, {"theta16": th16}
        ret, bcp, bcm = be.zeros(2 * P), be.zeros(P, B * N), be.zeros(P, B * N)
        folded = be.zeros(1) if centre_out else None
        order = dev(be, np.argsort(offs, kind="stable").astype(np.int32))
        if P:
            be.eval_mlp(dims, self.th, tb, dev(be, offs), order, P, sigma, self.ob, self.tg, ret[:P], ret[P:], bcp, bcm,
                        B, B * N, precision=mode, centre_out=folded, act=code, **self.kw)
        one, bc = be.zeros(1), be.zeros(B * N)
        be.eval_mlp_center(dims, self.th, self.ob, self.tg, one, bc, B, B * N, precision=mode, act=code, **self.ckw)
        torch.cuda.synchronize()
        self.ret = ret.double()
        self.Y = torch.cat([bcp, bcm, bc[None]]).view(2 * P + 1, B, N).double()   # [+..., -..., centre]
        self.centre_ret = float(one)
        self.folded = float(folded) if centre_out else None


def check_outputs(tag, mode, dims, code, run, theta, table, obs, tgt, offs, sigma):
    """Every output within its bound; the exact fp32 rows at the looser bar; every return within its reduction bound."""
    device = run.Y.device
    rows = tcm.form(mode, dims, theta, table, offs, sigma, centre=True, device=device)
    y, bound, exposed = tcm.forward(mode, rows, dims, tcm.layer0(mode, tcm.t64(obs, device)), code)
    assert torch.isfinite(run.Y).all(), f"{tag}: non-finite outputs"
    err = (run.Y - y).abs()
    worst = float((err / bound.clamp(min=1e-300)).max())
    bad = err > bound
    if bad.any():
        m, b, o = (int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{tag}: {int(bad.sum())} outputs beyond their bound, first member {m} row {b} output {o}: "
                             f"kernel {float(run.Y[m, b, o])!r}, model {float(y[m, b, o])!r}, bound {float(bound[m, b, o]):.3e}")
    exact = tcm.form(mode, dims, theta, table, offs, sigma, centre=True, device=device, exact=True)
    y64, b64 = tcm.bound_exact(mode, exact, dims, obs, code)
    worst64 = float(((run.Y - y64).abs() / b64.clamp(min=1e-300)).max())
    # returns from the kernel's own outputs
    r64, rb = tcm.returns64(run.Y, tcm.t64(tgt, device), code)
    P = len(offs)
    got = torch.cat([run.ret, torch.tensor([run.centre_ret], dtype=torch.float64, device=device)]) if P else \
        torch.tensor([run.centre_ret], dtype=torch.float64, device=device)
    rr = float(((got - r64).abs() / rb.clamp(min=1e-300)).max()) if float(rb.max()) > 0 else 0.0
    print(f"{tag}: worst error/bound {worst:.3f} ({int(exposed.sum())} of {exposed.numel()} outputs exposed to a "
          f"flip), vs exact fp32 rows {worst64:.3f}, returns {rr:.3f}")
    assert worst64 <= 1.0, f"{tag}: outputs beyond the bound from the exact fp32 rows ({worst64:.2f})"
    assert bool(((got - r64).abs() <= rb).all()), f"{tag}: a return is not its outputs' return ({rr:.2f})"
    if run.folded is not None:
        assert run.folded == run.centre_ret


# ------------------------------------------------------------------ every output of every member
# (dims, B, pairs): pairs such that the task groups (2 pairs chunks / 4) are at least twice the 33 clusters an
# H100's 132 SMs can hold
CLUSTER_SHAPES = {
    "one_layer": ([64, 32], 256, 40),                    # layer 0 is the last layer
    "widest_f16": ([256, 512, 512, 512], 256, 36),       # widest fp16 input, 4 N tiles per layer
    "bf16_wide_in": ([512, 512, 32], 256, 36),           # 512 inputs: the bf16 modes only
    "eight_narrow": ([64] * 8 + [32], 512, 24),          # 8 layers of one narrow tile each (even count)
    "odd_tiles": ([128, 384, 160], 768, 12),             # 3 + 2 = 5 tiles per task, B = 768
    "even_tiles": ([64, 256, 256], 512, 24),             # 2 + 2 tiles per task
}
DOMAINS = {"1x": (1.0, 1.0), "w8x": (8.0, 1.0), "obs255": (1.0, 255.0)}
TC_MODES = ("f16", "bf16", "bf16s")
# (shape, mode, code, domain, centre_out): two codes per shape and mode, one launch with the folded centre task and
# one without; then every code on the five-tile shape, alternating centre_out
CASES = []
for i, (name, (dims, B, pairs)) in enumerate(CLUSTER_SHAPES.items()):
    for j, mode in enumerate(TC_MODES):
        if mode == "f16" and name == "bf16_wide_in":
            continue
        for k in range(2):
            CASES.append((name, mode, CODES[(7 * i + 5 * j + 11 * k) % len(CODES)], list(DOMAINS)[(i + j + k) % 3],
                          k == 0))
CASES += [("odd_tiles", mode, c, "1x", i % 2 == 0) for mode in TC_MODES for i, c in enumerate(CODES)]


@pytest.mark.parametrize("shape,mode,code,domain,centre_out", CASES)
def test_every_output_and_return_within_bound_cluster_kernel(be, shape, mode, code, domain, centre_out):
    dims, B, pairs = CLUSTER_SHAPES[shape]
    assert (2 * pairs * B // 64) // 4 >= 2 * (be.sm_count // 4)
    w, o = DOMAINS[domain]
    theta, table, obs, tgt, offs = problem(dims, B, pairs, code, w_scale=w, obs_scale=o)
    sigma = 0.05
    run = Run(be, mode, dims, code, theta, table, obs, tgt, offs, sigma, centre_out=centre_out)
    check_outputs(f"{shape} {mode} {code:#x} {domain}", mode, dims, code, run, theta, table, obs, tgt, offs, sigma)


ANY_SHAPES = [([1, 17, 1], 63, 6), ([17, 127, 129], 65, 4), ([128, 129, 128], 255, 4), ([513, 64, 10], 1000, 2),
              ([3072, 128, 10], 64, 2), ([129, 513, 1], 1, 8), ([64, 128, 128], 256, 24)]


@pytest.mark.parametrize("i", range(len(ANY_SHAPES)))
def test_every_output_and_return_within_bound_f16_any(be, i):
    dims, B, pairs = ANY_SHAPES[i]
    code = CODES[(3 * i + 1) % len(CODES)]
    if mlp.decode(code)[2] != "mse" and dims[-1] == 1:
        code = mlp.code(mlp.decode(code)[0])
    theta, table, obs, tgt, offs = problem(dims, B, pairs, code, obs_scale=255.0 if i % 2 else 1.0)
    run = Run(be, "f16_any", dims, code, theta, table, obs, tgt, offs, 0.05)
    check_outputs(f"f16_any {dims} B={B} {code:#x}", "f16_any", dims, code, run, theta, table, obs, tgt, offs, 0.05)


# ------------------------------------------------------------------ the roundings, bit for bit
PIN = [("f16", [64, 512], 256), ("bf16", [64, 512], 256), ("bf16s", [64, 512], 256), ("f16_any", [64, 160], 256),
       ("f16_any", [63, 130], 255)]


def near_ties(rng, typ, n):
    """fp32 values within 3 fp32 ulps of a ``typ`` rounding tie, both signs, across magnitudes 2^-6 .. 2^6."""
    v = tcm.rn16(tcm.t64(rng.uniform(-1, 1, n) * 2.0 ** rng.randint(-6, 7, n)), typ)
    tie = v + tcm.spacing(v, typ) / 2 * torch.sign(v)
    t32 = tie.numpy().astype(np.float32)
    return (t32.view(np.int32) + rng.randint(-3, 4, n).astype(np.int32)).view(np.float32)


@pytest.mark.parametrize("mode,dims,B", PIN)
def test_one_hot_observations_pin_weight_formation(be, mode, dims, B):
    """Row b = e_(b mod K): y = fl32(W16[:, k] + b) for every member of both signs and the centre, bit for bit."""
    K, N = dims
    rng = np.random.RandomState(17)
    pairs = 24
    theta, table, _, _, offs = problem(dims, B, pairs)
    w = theta[: K * N]
    half = rng.rand(w.size) < 0.5
    w[half] = near_ties(rng, tcm.kind(mode), int(half.sum())) / 16
    theta[K * N:] = 0
    obs = np.zeros((B, K), np.float32)
    obs[np.arange(B), np.arange(B) % K] = 1
    tgt = np.zeros((B, N), np.float32)
    run = Run(be, mode, dims, 0, theta, table, obs, tgt, offs, 0.02)
    rows = tcm.form(mode, dims, theta, table, offs, 0.02, centre=True)
    W = rows[:, : K * N].view(-1, N, K)
    want = tcm.fl32(W[:, :, np.arange(B) % K].transpose(1, 2) + rows[:, K * N:][:, None, :])
    got = run.Y.cpu()
    diff = got != want
    assert not diff.any(), f"{int(diff.sum())} outputs differ, first at {diff.nonzero()[0].tolist()}: " \
                           f"{float(got[diff][0])!r} vs {float(want[diff][0])!r}"


def sweep(rng, typ, n):
    """Observations for the split: 0, +-2^-30 .. 2^-14 (x_lo subnormal or zero), values near 16-bit ties, ordinary
    values over 13 decades (16 in bf16), and 65504 .. 131023 (fp16 saturation of x_hi and of x_lo; bf16 up to 2^20).
    An fp16 observation of 131024 or more would enter as an infinity, and its row of identity outputs as NaN
    (inf * 0)."""
    big = np.array([65504, 65505, 65519, 65520, 65536, 1e5, 131008, 131009, 131023], np.float64)
    if typ == "bf16":                   # fp16: beyond 131023 x_lo is +-inf (test_infinite_observation_*)
        big = np.concatenate([big, [2 ** 17, 2 ** 20]])
    parts = [np.zeros(8), -np.zeros(8),
             rng.choice([-1, 1], n // 4) * 2.0 ** rng.uniform(-30, -14, n // 4),
             near_ties(rng, typ, n // 4) * 2.0 ** rng.randint(-8, 9, n // 4),
             rng.standard_normal(n // 4) * 10.0 ** rng.randint(-8, 8 if typ == "bf16" else 5, n // 4),
             1 + rng.randint(1, 4096, n // 8) * 2.0 ** -23, np.concatenate([big, -big])]
    x = np.concatenate(parts).astype(np.float32)
    return np.resize(rng.permutation(x), n)


def identity_theta(dims):
    return np.concatenate([np.concatenate([np.eye(m, k, dtype=np.float32).ravel(), np.zeros(m, np.float32)])
                           for k, m in zip(dims[:-1], dims[1:])])


def tie_close(a32, typ, ulps=2):
    """fp32 values within ``ulps`` fp32 ulps of a 16-bit rounding boundary (their rounding may differ between two
    libm implementations of the activation)."""
    lo, hi = a32.copy(), a32.copy()
    for _ in range(ulps):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
    return (tcm.rn16(tcm.t64(lo), typ) != tcm.rn16(tcm.t64(hi), typ)).numpy() & np.isfinite(a32)


@pytest.mark.parametrize("mode,dims,B", [(m, [64, 64], b) for m, b in (("f16", 256), ("bf16", 256), ("bf16s", 256),
                                                                         ("f16_any", 256), ("f16_any", 255))])
def test_identity_weights_pin_the_observation_split(be, mode, dims, B):
    """W = I, b = 0, the centre evaluation: y = fl32(x_hi + x_lo) in fp16, rn_bf16(x) in bf16, bit for bit."""
    obs = sweep(np.random.RandomState(3), tcm.kind(mode), B * dims[0]).reshape(B, dims[0])
    theta = identity_theta(dims)
    run = Run(be, mode, dims, 0, theta, np.zeros(64, np.float32), obs, np.zeros((B, dims[-1]), np.float32),
              np.zeros(0, np.int64), 0.0)
    ops = tcm.layer0(mode, obs)
    s = sum(ops)
    want = tcm.fl32(s)
    keep = (want == s).numpy()                          # the kernel adds x_hi and x_lo in fp32: exact sums only
    got = run.Y[0].cpu().numpy()
    print(f"{mode} B={B}: {int((~keep).sum())} of {keep.size} sums not exact in fp32, excluded")
    assert (~keep).sum() <= keep.size // 100
    np.testing.assert_array_equal(got[keep], want.numpy()[keep])


@pytest.mark.parametrize("hidden", list(mlp.HIDDEN_CODES))
@pytest.mark.parametrize("mode,B", [("f16", 256), ("bf16", 256), ("bf16s", 256), ("f16_any", 256), ("f16_any", 255)])
def test_two_identity_layers_pin_the_activation_rounding(be, hidden, mode, B):
    """Two identity layers: y = rn16(act(fl32(x_hi + x_lo))) for the hidden kind, bit for bit (signed zeros equal),
    except within 2 fp32 ulps of a 16-bit boundary, where numpy's libm may round its fp32 value differently."""
    dims = [64, 64, 64]
    typ = tcm.kind(mode)
    rng = np.random.RandomState(9)
    n = B * 64
    obs = np.concatenate([rng.uniform(-12, 12, n // 2), rng.standard_normal(n // 4) * 10.0 ** rng.randint(-4, 3, n // 4),
                          sweep(rng, typ, n - n // 2 - n // 4)]).astype(np.float32)
    obs = rng.permutation(obs).reshape(B, 64)
    code = mlp.code(hidden)
    run = Run(be, mode, dims, code, identity_theta(dims), np.zeros(64, np.float32), obs,
              np.zeros((B, 64), np.float32), np.zeros(0, np.int64), 0.0)
    y0 = tcm.fl32(sum(tcm.layer0(mode, obs))).numpy().astype(np.float32)
    with np.errstate(all="ignore"):
        a32 = orc.HIDDEN[hidden](y0).astype(np.float32)
    want = tcm.rn16(tcm.t64(a32), typ).numpy()
    s = sum(tcm.layer0(mode, obs))
    keep = ~tie_close(a32, typ) & (tcm.fl32(s) == s).numpy()
    got = run.Y[0].cpu().numpy()
    print(f"{hidden} {mode} B={B}: {int((~keep).sum())} of {keep.size} points within 2 fp32 ulps of a 16-bit tie, "
          f"excluded")
    # a sixteenth of the observations sits within 3 fp32 ulps of a 16-bit tie on purpose (the sweep)
    assert (~keep).sum() <= keep.size // 12
    assert (np.abs(want) == 65504).any() if typ == "f16" and hidden != "tanh" else True   # saturation reached
    np.testing.assert_array_equal(got[keep], want[keep])


# ------------------------------------------------------------------ row and member isolation, non-finite input
ISOLATION = [("f16", [128, 256, 64], 256), ("bf16", [128, 256, 64], 256), ("bf16s", [128, 256, 64], 256),
             ("f16_any", [100, 200, 10], 130)]


@pytest.mark.parametrize("mode,dims,B", ISOLATION)
def test_nan_observation_row_stays_in_its_row(be, mode, dims, B):
    theta, table, obs, tgt, offs = problem(dims, B, 6)
    clean = Run(be, mode, dims, 0, theta, table, obs, tgt, offs, 0.05).Y
    bad = obs.copy()
    r = B // 3
    bad[r, 1] = np.nan
    Y = Run(be, mode, dims, 0, theta, table, bad, tgt, offs, 0.05).Y
    assert torch.isnan(Y[:, r]).all()
    others = torch.ones(B, dtype=torch.bool)
    others[r] = False
    assert torch.equal(Y[:, others], clean[:, others])


@pytest.mark.parametrize("mode,B", [("f16", 256), ("f16_any", 255), ("bf16", 256), ("bf16s", 256)])
def test_infinite_observation_is_not_finite_in_any_precision(be, mode, B):
    """A one-layer policy on rows with +inf and -inf: the 16-bit evaluate gives the non-finite outputs the fp32
    evaluate gives (+-inf by the sign of the weight; NaN where the weight is 0), so a diverged member is not scored as
    a sane one.  fp16 takes a finite |x| up to 131023 (the x_hi + x_lo split saturates x_hi at 65504) and treats a
    larger one as the infinity of its sign; bf16 takes every finite value."""
    dims = [64, 32]
    theta, table, obs, tgt, offs = problem(dims, B, 4)
    theta[: 64 * 32].reshape(32, 64)[:4, 3] = 0            # the centre's exact zero weights give NaN, as in fp32
    obs[5, 3], obs[9, 7], obs[11, 3], obs[13, 3] = np.inf, -np.inf, 1e6, 131008.0
    Y = Run(be, mode, dims, 0, theta, table, obs, tgt, offs, 0.05).Y
    F = Run(be, "fp32", dims, 0, theta, table, obs, tgt, offs, 0.05).Y
    rows = [5, 9] + ([11] if tcm.kind(mode) == "f16" else [])
    inf_like = obs.copy()
    inf_like[11, 3] = np.inf
    Finf = Run(be, "fp32", dims, 0, theta, table, inf_like, tgt, offs, 0.05).Y
    for r in rows:
        for test in (torch.isposinf, torch.isneginf, torch.isnan):
            assert torch.equal(test(Y[:, r]), test(Finf[:, r])), (r, test.__name__)
    assert torch.isnan(Y[-1, 5, :4]).all() and not torch.isfinite(Y[:, 5]).any()
    fin = torch.ones(B, dtype=torch.bool)
    fin[rows] = False
    assert torch.isfinite(Y[:, fin]).all() and torch.isfinite(F[:, 11]).all()
