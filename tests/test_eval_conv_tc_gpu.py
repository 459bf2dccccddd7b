"""The tensor-core ("f16") evaluate of the conv + VirtualBatchNorm policy (examples/atari.py:14-37):
estk_eval_conv_vbn with ESTK_PREC_F16 against the reference golden, the CPU oracle's fp32 forward and the fp32
CUDA-core kernel, through the ctypes binding and through the public ES API.

Bar: every return within 1e-5 max-norm relative (SURVEY App. A.5) of the oracle's fp32 forward
of the materialised rows -- the same fp32-parity bar the MLP "f16" mode carries."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import es_oracle as orc
import estorch_b200 as E
from test_api_gpu import AtariPolicy

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def dev(be, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(be.device)


def _golden_frames():
    g = load_golden("atari_forward.npz")
    theta = g["theta16"].astype(np.float32)
    xref = g["xref8"].astype(np.float32) / np.float32(255)
    x = g["x8"].astype(np.float32) / np.float32(255)
    return g, theta, xref, x


def _table(rng, n, extra=1 << 12):
    """fp16-exact unit normals, like the engine's own table, and its exact fp16 copy."""
    table_len = (n + 31) // 32 * 32 + extra
    return orc.round_f16(rng.standard_normal(table_len).astype(np.float32))


def _run(be, precision, A, theta, table, offs, order, pairs, sigma, xref, obs, tgt, guard=0):
    """Returns of both kernels in one layout: [plus(pairs), minus(pairs)]; with guard > 0 the
    two return vectors sit inside NaN-filled guard bands that must stay untouched."""
    R, B = xref.shape[0], obs.shape[0]
    scratch = torch.empty(be.conv_scratch_bytes(R, B, precision), dtype=torch.uint8, device=be.device)
    kw = {}
    if precision == "f16" and offs is not None:
        tb16 = torch.from_numpy(table).to(torch.float16).to(be.device)
        assert np.array_equal(tb16.float().cpu().numpy(), table)
        kw["table16"] = tb16
    m = 1 if offs is None else pairs
    buf = torch.full((2 * guard + 2 * m + guard,), float("nan"), device=be.device)
    ret_p, ret_m = buf[guard: guard + m], buf[2 * guard + m: 2 * guard + 2 * m]
    be.eval_conv_vbn(A, dev(be, theta), None if table is None else dev(be, table), None if offs is None else dev(be, offs),
                     None if order is None else dev(be, order), pairs, sigma, dev(be, xref), dev(be, obs), dev(be, tgt),
                     ret_p, None if offs is None else ret_m, scratch, precision=precision, **kw)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    if guard:
        assert np.isnan(b[:guard]).all() and np.isnan(b[guard + m: 2 * guard + m]).all() and np.isnan(b[-guard:]).all()
    return np.concatenate([b[guard: guard + m], b[2 * guard + m: 2 * guard + 2 * m]]) if offs is not None else b[guard:guard + 1]


def _oracle(theta, table, offs, sigma, A, xref, obs, tgt, members=None):
    pop, _ = orc.sample_population(theta, table, offs, sigma)
    idx = range(pop.shape[0]) if members is None else members
    return np.array([orc.synthetic_return(orc.atari_forward(pop[i], A, xref, obs), tgt) for i in idx], np.float64)


# ------------------------------------------------------------------ 1. golden centre
def test_conv_f16_centre_matches_reference_golden(be):
    g, theta, xref, x = _golden_frames()
    A = 4
    tgt = np.random.RandomState(3).standard_normal((x.shape[0], A)).astype(np.float32)
    got = _run(be, "f16", A, theta, None, None, None, 1, 0.0, xref, x, tgt, guard=4)[0]
    want = float(orc.synthetic_return(g["logits"], tgt))       # logits from the unmodified reference
    f32 = _run(be, "fp32", A, theta, None, None, None, 1, 0.0, xref, x, tgt)[0]
    print(f"centre: f16 {got!r} fp32 kernel {f32!r} reference {want!r}")
    assert abs(got - want) < 2e-5 * abs(want)
    assert abs(got - f32) < 2e-5 * abs(f32)


# ------------------------------------------------------------------ 2. perturbed members vs the oracle
@pytest.mark.parametrize("frames", ["golden", "rand"])
def test_conv_f16_perturbed_members_vs_oracle(be, frames):
    g, theta, xref, x = _golden_frames()
    A, pairs, sigma = 4, 3, 0.02
    rng = np.random.RandomState(7)
    if frames == "rand":        # non-quantised frames: x_lo != 0
        gen = torch.Generator().manual_seed(11)
        xref = torch.rand(xref.shape, generator=gen).numpy()
        x = torch.rand(x.shape, generator=gen).numpy()
    tgt = rng.standard_normal((x.shape[0], A)).astype(np.float32)
    table = _table(rng, theta.size)
    offs = orc.noise_offsets(5, 0, 0, pairs, table.size, theta.size)
    want = _oracle(theta, table, offs, sigma, A, xref, x, tgt)
    got = _run(be, "f16", A, theta, table, offs, None, pairs, sigma, xref, x, tgt)
    f32 = _run(be, "fp32", A, theta, table, offs, None, pairs, sigma, xref, x, tgt)
    print(f"{frames}: f16 vs oracle {rel_err(got, want):.2e}, fp32 kernel vs oracle {rel_err(f32, want):.2e} (floor)")
    assert rel_err(got, want) < 1e-5


# ------------------------------------------------------------------ 3. shapes, order, guards; 5. determinism
@pytest.mark.parametrize("R,B,A,use_order", [(2, 1, 1, False), (5, 3, 18, True), (128, 32, 4, True),
                                             (130, 33, 64, False), (2, 33, 4, True), (130, 1, 1, True)])
def test_conv_f16_shapes_order_and_guards(be, R, B, A, use_order):
    rng = np.random.RandomState(R * 1000 + B * 10 + A)
    gen = torch.Generator().manual_seed(R + B + A)
    torch.manual_seed(R + B + A)
    m = AtariPolicy(A, None)
    theta = torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy().astype(np.float32)
    xref = torch.rand(R, 4, 84, 84, generator=gen).numpy()
    x = torch.rand(B, 4, 84, 84, generator=gen).numpy()
    tgt = rng.standard_normal((B, A)).astype(np.float32)
    pairs, sigma = 3, 0.02
    table = _table(rng, theta.size)
    offs = orc.noise_offsets(R + B, 1, 0, pairs, table.size, theta.size)
    order = np.argsort(offs, kind="stable").astype(np.int32)[::-1].copy() if use_order else None
    got = _run(be, "f16", A, theta, table, offs, order, pairs, sigma, xref, x, tgt, guard=8)
    again = _run(be, "f16", A, theta, table, offs, order, pairs, sigma, xref, x, tgt, guard=8)
    np.testing.assert_array_equal(got, again)                  # deterministic: no atomics
    want = _oracle(theta, table, offs, sigma, A, xref, x, tgt)  # member j at its own index, whatever the order
    f32 = _run(be, "fp32", A, theta, table, offs, order, pairs, sigma, xref, x, tgt)
    e16, e32 = rel_err(got, want), rel_err(f32, want)
    print(f"R={R} B={B} A={A} order={use_order}: f16 vs oracle {e16:.2e}, fp32 kernel vs oracle {e32:.2e}")
    # With two random reference frames some (c,h,w) variances are near zero and VBN divides by
    # them: returns reach -1e3 and the fp32 rounding of both kernels (and of the numpy oracle) is
    # amplified to ~1e-4.  The bar is 1e-5 or, where the fp32 kernel itself is that far off, 8x its
    # error (on an H100 the f16 kernel measured up to 1.7x for the population, 5.0x for the centre).
    assert e16 < max(1e-5, 8 * e32)
    centre = _run(be, "f16", A, theta, None, None, None, 1, 0.0, xref, x, tgt, guard=8)[0]
    c32 = _run(be, "fp32", A, theta, None, None, None, 1, 0.0, xref, x, tgt)[0]
    wc = float(orc.synthetic_return(orc.atari_forward(theta, A, xref, x), tgt))
    assert abs(centre - wc) < max(1e-5, 8 * abs(c32 - wc) / abs(wc)) * abs(wc)


# ------------------------------------------------------------------ 4. full size
def test_conv_f16_full_size_vs_fp32_kernel_and_oracle(be):
    """BASELINE config 5: P = 1024, R = 128, B = 32, A = 4.  All 1024 returns against the fp32
    kernel; 16 sampled members against the oracle; what the difference does to the ranks."""
    A, R, B, P, sigma = 4, 128, 32, 1024, 0.02
    pairs = P // 2
    torch.manual_seed(0)
    m = AtariPolicy(A, None)
    theta = torch.nn.utils.parameters_to_vector(m.parameters()).detach().contiguous()
    n = theta.numel()
    gen = torch.Generator().manual_seed(1234)
    xref, x = torch.rand(R, 4, 84, 84, generator=gen), torch.rand(B, 4, 84, 84, generator=gen)
    tgt = torch.randn(B, A, generator=gen)
    table = be.alloc(1 << 24)
    be.fill_noise_table(table, 42)
    tb16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, tb16) == 0
    offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
    th_d, xr_d, x_d, t_d = theta.to(be.device), xref.to(be.device), x.to(be.device), tgt.to(be.device)
    res = {}
    for mode in ("fp32", "f16", "f16"):
        scratch = torch.empty(be.conv_scratch_bytes(R, B, mode), dtype=torch.uint8, device=be.device)
        r = be.zeros(P)
        be.eval_conv_vbn(A, th_d, table, offs, order, pairs, sigma, xr_d, x_d, t_d, r[:pairs], r[pairs:], scratch,
                         precision=mode, table16=tb16 if mode == "f16" else None)
        torch.cuda.synchronize()
        if mode in res:
            assert torch.equal(res[mode], r)                    # bit-identical run to run
        res[mode] = r
        del scratch
    f32, f16 = res["fp32"].cpu().numpy(), res["f16"].cpu().numpy()
    sample = np.linspace(0, P - 1, 16).round().astype(int)
    tab_h, offs_h = table.cpu().numpy(), offs.cpu().numpy()
    want = np.empty(len(sample))
    for i, mbr in enumerate(sample):
        j = mbr % pairs
        pop, _ = orc.sample_population(theta.numpy(), tab_h, offs_h[j:j + 1], sigma)
        want[i] = orc.synthetic_return(orc.atari_forward(pop[0 if mbr < pairs else 1], A, xref.numpy(), x.numpy()),
                                       tgt.numpy())
    e16, e32 = rel_err(f16[sample], want), rel_err(f32[sample], want)
    all_diff = rel_err(f16, f32)
    r16, r32 = orc.compute_ranks(f16), orc.compute_ranks(f32)
    d = np.abs(r16.astype(np.int64) - r32)
    print(f"full size: f16 vs oracle {e16:.2e}, fp32 kernel vs oracle {e32:.2e}, f16 vs fp32 kernel (all {P}) "
          f"{all_diff:.2e}; rank indices differing {int(np.count_nonzero(d))}, mean displacement {d.mean():.3f}, "
          f"max {int(d.max())}")
    assert e16 < 1e-5
    # the two kernels differ by no more than each one's distance from the oracle allows
    assert all_diff < 1e-5 + 2 * e32
    assert d.mean() < 8


# ------------------------------------------------------------------ 6. public API
def _atari_setup():
    g = torch.Generator().manual_seed(5)
    xref = torch.rand(8, 4, 84, 84, generator=g)
    obs, tgt = torch.rand(4, 4, 84, 84, generator=g), torch.randn(4, 4, generator=g)
    return xref, obs, tgt


def test_conv_f16_fused_generation_vs_oracle():
    xref, obs, tgt = _atari_setup()
    rec = {}

    class Q(E.ES):
        def log(self):
            rec["returns"] = self.population_returns[:, 0].copy()
            rec["episode"] = self.episode_reward
    torch.manual_seed(1)
    P, sigma, table_len, seed = 8, 0.02, 1 << 21, 9
    es = Q(AtariPolicy, E.DeviceAgent, torch.optim.Adam, population_size=P, sigma=sigma,
           policy_kwargs=dict(n_actions=4, xref=xref), agent_kwargs=dict(obs=obs, target=tgt),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=table_len, noise_seed=seed, eval_precision="f16")
    assert es._fused and es._is_conv and es._precision == "f16"
    theta0 = es._slots[0].theta.cpu().numpy().copy()
    table = es._table.cpu().numpy()
    es.train(n_steps=1)
    n = theta0.size
    offs = orc.noise_offsets(seed, 0, 0, P // 2, table_len, n)
    pop, eps = orc.sample_population(theta0, table, offs, sigma)
    want = np.array([orc.synthetic_return(orc.atari_forward(pop[i], 4, xref.numpy(), obs.numpy()), tgt.numpy())
                     for i in range(P)])
    assert rel_err(rec["returns"], want) < 1e-5
    np.testing.assert_array_equal(es._ranks.cpu().numpy(), orc.compute_ranks(rec["returns"]))
    grad = orc.calculate_grad(rec["returns"], eps, sigma)
    assert rel_err(es._grad.cpu().numpy(), grad) < 1e-5
    th, _, _ = orc.adam_step(theta0, np.zeros(n, np.float32), np.zeros(n, np.float32),
                             orc.negate_clamp(es._grad.cpu().numpy()), 1)
    assert rel_err(es._slots[0].theta.cpu().numpy(), th) < 1e-6
    ep = float(orc.synthetic_return(orc.atari_forward(th, 4, xref.numpy(), obs.numpy()), tgt.numpy()))
    assert abs(rec["episode"] - ep) < 1e-5 * abs(ep)


def test_conv_f16_graph_replay_equals_eager(monkeypatch):
    xref, obs, tgt = _atari_setup()
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ESTORCH_B200_GRAPH", mode)
        torch.manual_seed(4)
        es = E.ES(AtariPolicy, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.02,
                  policy_kwargs=dict(n_actions=4, xref=xref), agent_kwargs=dict(obs=obs, target=tgt),
                  optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 21, eval_precision="f16")
        es.log = lambda: None
        es.train(n_steps=7)
        s = es._slots[0]
        out[mode] = (s.theta.clone(), s.m.clone(), s.v.clone(), s.best_theta.clone(), es.episode_reward,
                     es.best_reward, sum(isinstance(v, tuple) for v in es.__dict__.get("_graphs", {}).values()))
    a, b = out["1"], out["0"]
    assert a[6] >= 1 and b[6] == 0                       # graphs were actually used / not used
    for x, y in zip(a[:4], b[:4]):
        assert torch.equal(x, y)
    assert a[4] == b[4] and a[5] == b[5]


@pytest.mark.parametrize("precision", ["bf16", "bf16s"])
def test_conv_policy_rejects_bf16_modes(precision):
    xref, obs, tgt = _atari_setup()
    with pytest.raises(ValueError, match="'fp32' and 'f16'"):
        E.ES(AtariPolicy, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.02,
             policy_kwargs=dict(n_actions=4, xref=xref), agent_kwargs=dict(obs=obs, target=tgt),
             optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 21, eval_precision=precision)


def test_conv_policy_auto_stays_fp32():
    xref, obs, tgt = _atari_setup()
    es = E.ES(AtariPolicy, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.02,
              policy_kwargs=dict(n_actions=4, xref=xref), agent_kwargs=dict(obs=obs, target=tgt),
              optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 21)
    assert es._fused and es._precision == "fp32"
