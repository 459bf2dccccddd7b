"""Cross-entropy objective (include/estk.h ESTK_LOSS_XENT) on the H100: the fp32 and wgmma MLP evaluate
kernels against the fp64 cross-entropy of the oracle's forwards (tests/_xent_oracle.py), run-to-run
bit equality, large logits, refused codes, ES / NSR-ES against the reference-generated goldens, and the
north-star accuracy that ``eval_precision="auto"`` rests on."""
import json

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import es_oracle as orc
import _xent_oracle as xo
from _xent_oracle import MLP, XENT_ACTS, XentOracleBackend
from test_eval_mlp_act_gpu import _eval, _set_theta, _tc_problem, dev
import estorch_b200 as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def _soft_targets(rng, B, C, onehot=False):
    if onehot:
        return np.eye(C, dtype=np.float32)[rng.randint(0, C, B)]
    return rng.dirichlet(np.ones(C), B).astype(np.float32)


def _twice(be, *args, **kw):
    """Two identical launches: the returns (and BCs, centre) must be the same bits."""
    a = _eval(be, *args, **kw)
    b = _eval(be, *args, **kw)
    np.testing.assert_array_equal(a[0], b[0])
    if a[1] is not None:
        np.testing.assert_array_equal(a[1], b[1])
    assert a[2] == b[2] or (a[2] is None and b[2] is None)
    return a


# ------------------------------------------------------------------ fp32 CUDA-core kernel
@pytest.mark.parametrize("code", XENT_ACTS)
@pytest.mark.parametrize("dims,B,pairs,bc", [([4, 64, 64, 3], 256, 8, 0), ([784, 100, 10], 100, 4, 0),
                                              ([32, 64, 64, 64, 64, 64, 64, 64, 10], 70, 3, 0),
                                              ([24, 64, 64, 4], 256, 4, 256)])
def test_fp32_xent_vs_oracle(be, dims, B, pairs, bc, code):
    hidden = xo.hidden_of(code)
    rng = np.random.RandomState(7)
    n = orc.mlp_param_count(dims)
    table_len = max(1 << 14, (n + 31) // 32 * 32 + 4096)
    table = rng.standard_normal(table_len).astype(np.float32)
    theta = (rng.standard_normal(n) * 0.1).astype(np.float32)
    obs = rng.standard_normal((B, dims[0])).astype(np.float32)
    tgt = _soft_targets(rng, B, dims[-1], onehot=(dims[-1] == 10))
    offs = orc.noise_offsets(5, 0, 0, pairs, table_len, n)
    ret, bcs, _ = _twice(be, dims, theta, table, offs, 0.02, obs, tgt, code, 64 if bc else 0, bc)
    pop, _ = orc.sample_population(theta, table, offs, 0.02)
    want, want_bc = xo.evaluate_population(pop, dims, obs, tgt, 64 if bc else 0, bc, hidden)
    assert rel_err(ret, want) < 2e-6
    if bc:
        assert rel_err(bcs, want_bc) < 2e-6
    one = be.zeros(1)
    be.eval_mlp_center(dims, dev(be, theta), dev(be, obs), dev(be, tgt), one, act=code)
    w = float(xo.xent_return(xo.forward(theta, dims, obs, hidden), tgt))
    assert abs(float(one) - w) < 2e-6 * abs(w)


# ------------------------------------------------------------------ wgmma kernel
TC_TOL = {"f16": (1e-5, 3e-5, 2e-3), "bf16": (5e-4, 2e-2, 5e-3), "bf16s": (5e-4, 3e-2, 5e-3)}
# the last layer's N tiles: one narrow tile of 32, one, two, 2 * 128 + 32, three, four
TILE_DIMS = [[64, 32], [64, 128, 128], [64, 256, 256], [128, 256, 288], [64, 128, 384], [64, 512, 512]]


def _tc_kw(be, mode, theta, table):
    th, tb = dev(be, theta), dev(be, table)
    kw = {}
    if mode == "f16":
        kw["table16"] = be.alloc(table.size, dtype=torch.float16)
        assert be.shadow_f16(tb, kw["table16"]) == 0
    elif mode == "bf16s":
        kw["theta16"], kw["table16"] = be.alloc(theta.size, dtype=torch.bfloat16), be.alloc(table.size,
                                                                                          dtype=torch.bfloat16)
        be.shadow_bf16(th, kw["theta16"])
        be.shadow_bf16(tb, kw["table16"])
    return kw


@pytest.mark.parametrize("code", XENT_ACTS)
@pytest.mark.parametrize("mode", ["f16", "bf16", "bf16s"])
@pytest.mark.parametrize("dims", TILE_DIMS)
def test_tensor_core_xent_vs_emulation_and_fp32(be, dims, mode, code):
    hidden = xo.hidden_of(code)
    B, pairs, bc = 512, 3, 256
    n, table, theta, obs, _, offs = _tc_problem(dims, B, pairs)
    tgt = _soft_targets(np.random.RandomState(len(dims) + dims[-1]), B, dims[-1])
    assert be.eval_supports_f16(dims, B, act=code) and be.eval_supports_bf16(dims, B, act=code)
    kw = _tc_kw(be, mode, theta, table)
    got, got_bc, centre = _twice(be, dims, theta, table, offs, 0.02, obs, tgt, code, 64, bc, precision=mode,
                                 centre=True, **kw)
    emu_be = XentOracleBackend(tensor_core=True)
    rows = emu_be._rows(torch.from_numpy(theta), torch.from_numpy(table), torch.from_numpy(offs), 0.02, dims, mode)
    emu, emu_bc = xo.evaluate_population(rows, dims, obs, tgt, 64, bc, hidden, precision=mode)
    pop, _ = orc.sample_population(theta, table, offs, 0.02)
    exact, _ = xo.evaluate_population(pop, dims, obs, tgt, 64, bc, hidden)
    t_emu, t_exact, t_bc = TC_TOL[mode]
    print(f"{mode} act={code:#x} {dims}: vs emulation {rel_err(got, emu):.2e}, vs fp32 {rel_err(got, exact):.2e}")
    assert rel_err(got, emu) < t_emu
    assert rel_err(got, exact) < t_exact
    assert rel_err(got_bc, emu_bc) < t_bc
    # the folded centre task and the centre call (offsets NULL) evaluate theta itself: the same bits
    one = be.zeros(1)
    be.eval_mlp_center(dims, dev(be, theta), dev(be, obs), dev(be, tgt), one, precision=mode, act=code,
                       **({"theta16": kw["theta16"]} if mode == "bf16s" else {}))
    ct = torch.zeros(1)
    emu_be.eval_mlp_center(dims, torch.from_numpy(theta), torch.from_numpy(obs), torch.from_numpy(tgt), ct,
                           precision=mode, act=code)
    assert abs(float(one) - float(ct)) < t_emu * abs(float(ct))
    assert centre == float(one)


@pytest.mark.parametrize("mode", ["fp32", "f16"])
def test_large_logits_stay_finite_and_match_fp64(be, mode):
    """|y| ~ 200: exp(y) overflows fp32 without the max shift."""
    dims, B, pairs = [64, 128, 64], 256, 2
    n, table, theta, obs, _, offs = _tc_problem(dims, B, pairs, seed=5)
    theta = theta.copy()
    w2 = dims[0] * dims[1] + dims[1]
    theta[w2:] *= 400.0                                          # the last layer's weights and biases
    tgt = _soft_targets(np.random.RandomState(9), B, dims[-1])
    kw = _tc_kw(be, mode, theta, table) if mode != "fp32" else {}
    got, _, _ = _twice(be, dims, theta, table, offs, 0.001, obs, tgt, xo.LOSS_XENT, precision=mode, **kw)
    rows = XentOracleBackend(tensor_core=True)._rows(torch.from_numpy(theta), torch.from_numpy(table),
                                                     torch.from_numpy(offs), 0.001, dims, mode)
    logits = xo.forward(rows[0], dims, obs, "relu", mode)
    assert 100 < np.abs(logits).max() < 1000
    want, _ = xo.evaluate_population(rows, dims, obs, tgt, precision=mode)
    assert np.all(np.isfinite(got))
    print(f"large logits {mode}: max |y| {np.abs(logits).max():.1f}, vs fp64 {rel_err(got, want):.2e}")
    assert rel_err(got, want) < 1e-5


def test_refused_codes_return_before_launch_and_leave_the_returns(be):
    dims, B = [64, 64, 32], 256
    n, table, theta, obs, tgt, offs = _tc_problem(dims, B, 2)
    for code in (0x10101, 0x20000, 0x10200, 0x10100):
        ret = torch.full((4,), 7.0, device=be.device)
        args = (dev(be, theta), dev(be, table), dev(be, offs), None, 2, 0.02, dev(be, obs), dev(be, tgt),
                ret[:2], ret[2:])
        with pytest.raises(RuntimeError, match=r"estk_status -1\)"):                  # ESTK_ERR_INVALID
            be.eval_mlp(dims, *args, act=code)
        for mode in ("f16", "bf16"):
            with pytest.raises(RuntimeError, match="not supported"):                  # ESTK_ERR_UNSUPPORTED
                be.eval_mlp(dims, *args, act=code, precision=mode, **_tc_kw(be, mode, theta, table))
        torch.cuda.synchronize()
        assert torch.equal(ret.cpu(), torch.full((4,), 7.0))
    # a 10-class head is not a tensor-core shape: refused there, evaluated by the fp32 kernel
    assert not be.eval_supports_f16([64, 64, 10], B, act=xo.LOSS_XENT)


# ------------------------------------------------------------------ public API vs the reference goldens
def test_es_fused_xent_vs_reference_golden():
    g = load_golden("es_xent_p64.npz")
    dims = [int(d) for d in g["dims"]]
    rec = []

    class R(E.ES):
        def log(self):
            rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                            best=self.best_reward))
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.1, policy_kwargs={"dims": dims},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]),
                             loss="cross_entropy"),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]))
    assert es._fused and es._be.name == "cuda" and es._act_code() == xo.LOSS_XENT
    es._table.copy_(torch.from_numpy(g["table"]))
    _set_theta(es.policy, g["theta0"])
    es.train(n_steps=3)
    for gen in range(3):
        assert rel_err(rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-5
        assert abs(rec[gen]["episode"] - float(g["episode_reward"][gen])) < 2e-5
        assert abs(rec[gen]["best"] - float(g["best_reward"][gen])) < 2e-5
    theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().cpu().numpy()
    assert rel_err(theta, g["theta_after"][2]) < 2e-4


def test_nsr_fused_xent_vs_reference_golden():
    g = load_golden("nsr_xent_p32.npz")
    dims = [int(d) for d in g["dims"]]
    rec = []

    class R(E.NSR_ES):
        def log(self):
            rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward, idx=self.idx))
    np.random.seed(123)
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=32, sigma=0.02, policy_kwargs={"dims": dims},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]), bc_obs=64,
                             bc_dim=256, loss="cross_entropy"),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]))
    assert es._fused and es._be.name == "cuda"
    es._table.copy_(torch.from_numpy(g["table"]))
    for i, (p, _) in enumerate(es.meta_population):
        _set_theta(p, g["meta_theta0"][i])
        es._slots[i].push_theta()
    es._archive = [a.copy() for a in g["archive0"]]
    np.random.seed(123)
    es.train(n_steps=len(g["grad"]))
    for gen in range(len(g["grad"])):
        assert rec[gen]["idx"] == int(g["idx"][gen])
        assert rel_err(rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-4
        assert rel_err(rec[gen]["returns"][:, 1], g["returns"][gen][:, 1]) < 1e-4
        assert abs(rec[gen]["episode"] - float(g["episode_reward"][gen])) < 1e-4
    np.testing.assert_allclose(np.stack(es._archive), g["archive_final"], rtol=1e-3, atol=1e-4)


def test_auto_picks_f16_for_a_tensor_core_cross_entropy_shape_and_trains():
    rng = np.random.RandomState(4)
    dims, B = [64, 128, 64], 256
    obs = torch.from_numpy(rng.standard_normal((B, 64)).astype(np.float32))
    tgt = torch.from_numpy(_soft_targets(rng, B, 64, onehot=True))
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=256, sigma=0.02, policy_kwargs={"dims": dims},
              agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy"), optimizer_kwargs={"lr": 0.01})
    es.log = lambda: None
    assert es._fused and es._precision == "f16"
    es.train(n_steps=4)
    with torch.no_grad():
        want = -float(torch.nn.functional.cross_entropy(es.policy(obs.to(es._dev)), tgt.to(es._dev)))
    assert abs(es.episode_reward - want) < 1e-4 * abs(want)


# ------------------------------------------------------------------ north star: the evidence for "auto"
def test_north_star_xent_accuracy_per_mode(be):
    """P = 4096, B = 256, the north-star body with a 256-class head: 512 members (the + and - of 256
    pairs) of every evaluate precision against the CPU fp32 forward (max-norm relative)."""
    dims = [128, 512, 512, 512, 512, 256]
    n, P, pairs, sigma = orc.mlp_param_count(dims), 4096, 2048, 0.02
    torch.manual_seed(0)
    mods = []
    for i in range(len(dims) - 1):
        l = torch.nn.Linear(dims[i], dims[i + 1])
        mods += [l.weight.detach().reshape(-1), l.bias.detach()]
    theta = torch.cat(mods).contiguous()
    g = torch.Generator().manual_seed(1234)
    obs = torch.randn(256, 128, generator=g)
    tgt = torch.nn.functional.one_hot(torch.randint(0, 256, (256,), generator=g), 256).to(torch.float32)
    table = be.alloc(1 << 26)
    be.fill_noise_table(table, 42)
    offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
    th_d, obs_d, tgt_d = theta.to(be.device), obs.to(be.device), tgt.to(be.device)
    tb16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, tb16) == 0
    th16, tbb = be.alloc(n, dtype=torch.bfloat16), be.alloc(table.numel(), dtype=torch.bfloat16)
    be.shadow_bf16(th_d, th16)
    be.shadow_bf16(table, tbb)
    extra = {"fp32": {}, "f16": {"table16": tb16}, "bf16": {}, "bf16s": {"theta16": th16, "table16": tbb}}
    res = {}
    for mode in ("fp32", "f16", "bf16", "bf16s"):
        r = be.zeros(P)
        be.eval_mlp(dims, th_d, table, offs, order, pairs, sigma, obs_d, tgt_d, r[:pairs], r[pairs:], precision=mode,
                    act=xo.LOSS_XENT, **extra[mode])
        res[mode] = r.cpu().numpy()
    tab_h, offs_h, th_h = table.cpu().numpy(), offs.cpu().numpy(), theta.numpy()
    sel = np.arange(0, pairs, pairs // 256)
    want_p, want_m = [], []
    for c in range(0, sel.size, 32):
        pop, _ = orc.sample_population(th_h, tab_h, offs_h[sel[c: c + 32]], sigma)
        w, _ = xo.evaluate_population(pop, dims, obs.numpy(), tgt.numpy())
        want_p.append(w[:len(w) // 2])
        want_m.append(w[len(w) // 2:])
    want = np.concatenate(want_p + want_m)
    idx = np.concatenate([sel, pairs + sel])
    report = {"dims": dims, "members_compared": int(idx.size)}
    for mode in res:
        report[f"{mode}_max_rel_err"] = rel_err(res[mode][idx], want)
    print("NORTH_STAR_XENT " + json.dumps(report))
    assert report["fp32_max_rel_err"] < 2e-6
    assert report["f16_max_rel_err"] < 1e-5          # eval_precision="auto" picks f16 for the cross-entropy
    assert report["bf16_max_rel_err"] < 2e-2 and report["bf16s_max_rel_err"] < 3e-2
