"""ELU, SiLU and LeakyReLU MLP policies on the H100: the nine new activation codes of include/estk.h
in every MLP evaluate kernel (fp32 shared-memory, fp32 streamed, f16 / bf16 / bf16s cluster, f16_any
streamed) against the oracle emulations of tests/_mlp_oracle.py and the exact fp32 forward;
determinism; large pre-activations; the north-star shape per kind; and ES / NSR-ES runs against the
reference-generated goldens."""
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden, rel_err
from oracle import es_oracle as orc
import _mlp_oracle as mlp
from _mlp_oracle import MLP, NEW_ACTS, decode
from _oracle_backend import OracleBackend
import estorch_b200 as E

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


def _problem(dims, B, pairs, loss, seed=23):
    rng = np.random.RandomState(seed)
    n = orc.mlp_param_count(dims)
    table_len = (n + 31) // 32 * 32 + (1 << 14)
    table = orc.round_f16(rng.standard_normal(table_len).astype(np.float32))   # fp16-exact, like the engine's
    theta = np.concatenate([np.concatenate([(rng.uniform(-1, 1, dims[i] * dims[i + 1]) / np.sqrt(dims[i])),
                                            rng.uniform(-1, 1, dims[i + 1]) / np.sqrt(dims[i])])
                            for i in range(len(dims) - 1)]).astype(np.float32)
    obs = rng.standard_normal((B, dims[0])).astype(np.float32)
    if loss == "xent":
        tgt = np.eye(dims[-1], dtype=np.float32)[rng.randint(0, dims[-1], B)]
    else:
        tgt = rng.uniform(-0.9, 0.9, (B, dims[-1])).astype(np.float32)
    offs = orc.noise_offsets(11, 0, 0, pairs, table_len, n)
    return n, table, theta, obs, tgt, offs


def _tables(be, table, theta, mode):
    th, tb, kw = dev(be, theta), dev(be, table), {}
    if mode in ("f16", "f16_any"):
        kw["table16"] = be.alloc(table.size, dtype=torch.float16)
        assert be.shadow_f16(tb, kw["table16"]) == 0
    elif mode == "bf16s":
        kw["theta16"], kw["table16"] = be.alloc(theta.size, dtype=torch.bfloat16), be.alloc(table.size, dtype=torch.bfloat16)
        be.shadow_bf16(th, kw["theta16"])
        be.shadow_bf16(tb, kw["table16"])
    return th, tb, kw


def _eval(be, dims, th, tb, offs, sigma, obs, tgt, code, mode, kw, bc_obs=0, bc_dim=0, order=True, centre=False):
    pairs = len(offs)
    ret = be.zeros(2 * pairs)
    bcp = be.zeros(pairs, bc_dim) if bc_dim else None
    bcm = be.zeros(pairs, bc_dim) if bc_dim else None
    c_out = be.zeros(1) if centre else None
    o = dev(be, np.argsort(offs, kind="stable").astype(np.int32)) if order else None
    be.eval_mlp(dims, th, tb, dev(be, offs), o, pairs, sigma, dev(be, obs), dev(be, tgt), ret[:pairs], ret[pairs:],
                bcp, bcm, bc_obs, bc_dim, precision=mode, centre_out=c_out, act=code, **kw)
    torch.cuda.synchronize()
    bcs = None if not bc_dim else np.concatenate([bcp.cpu().numpy(), bcm.cpu().numpy()])
    return ret.cpu().numpy(), bcs, (None if c_out is None else float(c_out))


def _want(dims, theta, table, offs, obs, tgt, code, mode, bc_obs=0, bc_dim=0):
    if mode == "fp32":
        rows, _ = orc.sample_population(theta, table, offs, 0.02)
    else:
        rows = OracleBackend(tensor_core=True)._rows(torch.from_numpy(theta), torch.from_numpy(table),
                                                     torch.from_numpy(offs), 0.02, dims, mode)
    return mlp.evaluate_population(rows, dims, obs, tgt, code, mode, bc_obs, bc_dim)


# ------------------------------------------------------------------ fp32 CUDA-core kernels
# ([17, 33, 5], 100): the shared-memory kernel; [64, 1200, 10]: a layer too wide for it (streamed);
# ([4, 64, 2], 40000): more than 64 observation chunks (streamed)
@pytest.mark.parametrize("code", NEW_ACTS)
@pytest.mark.parametrize("dims,B,pairs", [([17, 33, 5], 100, 6), ([9, 130, 70, 70, 3], 256, 3),
                                          ([64, 1200, 10], 70, 2), ([4, 64, 2], 40000, 2)])
def test_fp32_kernels_vs_oracle(be, dims, B, pairs, code):
    hidden, output, loss = decode(code)
    n, table, theta, obs, tgt, offs = _problem(dims, B, pairs, loss)
    th, tb, kw = _tables(be, table, theta, "fp32")
    bc_dim = 16 * dims[-1]
    ret, bcs, _ = _eval(be, dims, th, tb, offs, 0.02, obs, tgt, code, "fp32", kw, 16, bc_dim)
    want, want_bc = _want(dims, theta, table, offs, obs, tgt, code, "fp32", 16, bc_dim)
    assert rel_err(ret, want) < 5e-6
    assert rel_err(bcs, want_bc) < 5e-6
    one = be.zeros(1)
    be.eval_mlp_center(dims, th, dev(be, obs), dev(be, tgt), one, act=code)
    w = float(mlp.member_return(orc.mlp_forward(theta, dims, obs, hidden, output), tgt, loss))
    assert abs(float(one) - w) < 5e-6 * abs(w) + 1e-7


# ------------------------------------------------------------------ tensor-core kernels
# per mode: (vs its emulation, vs the exact fp32 forward, BC vs emulation) -- the ReLU and Tanh tests' bars
TC_TOL = {"f16": (1e-5, 3e-5, 2e-3), "f16_any": (1e-5, 3e-5, 2e-3), "bf16": (5e-4, 2e-2, 5e-3),
          "bf16s": (5e-4, 3e-2, 5e-3)}


@pytest.mark.parametrize("code", NEW_ACTS)
@pytest.mark.parametrize("mode,dims,B,pairs", [("f16", [64, 256, 64], 512, 4), ("bf16", [64, 256, 64], 512, 4),
                                               ("bf16s", [64, 256, 64], 512, 4),
                                               ("f16", [128, 512, 512, 288], 256, 3),
                                               ("f16_any", [33, 200, 70, 10], 100, 3),
                                               ("f16_any", [784, 256, 10], 300, 2)])
def test_tensor_core_modes_vs_emulation_and_fp32(be, mode, dims, B, pairs, code):
    hidden, output, loss = decode(code)
    n, table, theta, obs, tgt, offs = _problem(dims, B, pairs, loss)
    if mode == "f16_any":
        assert not be.eval_supports_f16(dims, B, act=code) and be.eval_supports_f16_any(dims, B, act=code)
    else:
        assert be.eval_supports_f16(dims, B, act=code) and be.eval_supports_bf16(dims, B, act=code)
    th, tb, kw = _tables(be, table, theta, mode)
    bc_dim = 256 if dims[-1] >= 64 else 64
    centre = mode != "f16_any"
    got, got_bc, c_fold = _eval(be, dims, th, tb, offs, 0.02, obs, tgt, code, mode, kw, 64, bc_dim, centre=centre)
    emu, emu_bc = _want(dims, theta, table, offs, obs, tgt, code, mode, 64, bc_dim)
    exact, exact_bc = _want(dims, theta, table, offs, obs, tgt, code, "fp32", 64, bc_dim)
    t_emu, t_exact, t_bc = TC_TOL[mode]
    print(f"{mode} act={code:#x} {dims}: vs emulation {rel_err(got, emu):.2e}, vs fp32 {rel_err(got, exact):.2e}")
    assert rel_err(got, emu) < t_emu
    assert rel_err(got, exact) < t_exact
    assert rel_err(got_bc, emu_bc) < t_bc
    if mode in ("f16", "f16_any"):
        assert rel_err(got_bc, exact_bc) < 2e-3
    # bits repeat from launch to launch, with and without the evaluation order
    again, again_bc, _ = _eval(be, dims, th, tb, offs, 0.02, obs, tgt, code, mode, kw, 64, bc_dim, order=False,
                               centre=centre)
    np.testing.assert_array_equal(got, again)
    np.testing.assert_array_equal(got_bc, again_bc)
    # the centre call evaluates theta itself; the folded centre task gives the same bits
    one = be.zeros(1)
    be.eval_mlp_center(dims, th, dev(be, obs), dev(be, tgt), one, precision=mode, act=code,
                       **({"theta16": kw["theta16"]} if mode == "bf16s" else {}))
    ct = torch.zeros(1)
    OracleBackend(tensor_core=True).eval_mlp_center(dims, torch.from_numpy(theta), torch.from_numpy(obs),
                                                          torch.from_numpy(tgt), ct, precision=mode, act=code)
    assert abs(float(one) - float(ct)) < t_emu * abs(float(ct))
    if centre:
        assert c_fold == float(one)


def test_fp32_repeats_bit_for_bit_with_and_without_order(be):
    for code in NEW_ACTS:
        dims, B, pairs = [17, 100, 10], 300, 5
        n, table, theta, obs, tgt, offs = _problem(dims, B, pairs, decode(code)[2])
        th, tb, kw = _tables(be, table, theta, "fp32")
        a = _eval(be, dims, th, tb, offs, 0.02, obs, tgt, code, "fp32", kw, 8, 80)
        b = _eval(be, dims, th, tb, offs, 0.02, obs, tgt, code, "fp32", kw, 8, 80, order=False)
        np.testing.assert_array_equal(a[0], b[0])
        np.testing.assert_array_equal(a[1], b[1])


# ------------------------------------------------------------------ large pre-activations
# y = x exactly: identity weights, zero biases, so the behaviour characteristic is act(x) itself
XS = np.float32([-1e4, -100.0, -90.0, -89.0, -88.5, -50.0, -17.0, -1.0, -0.125, -0.0, 0.0, 0.125, 1.0, 17.0,
                 50.0, 100.0, 6e4, 7e4])


@pytest.mark.parametrize("mode", ["fp32", "f16", "bf16"])
@pytest.mark.parametrize("hidden", mlp.NEW_KINDS)
def test_large_preactivations_are_finite_and_exact(be, hidden, mode):
    dims, B = [64, 64, 64], 256
    eye = np.eye(64, dtype=np.float32)
    theta = np.concatenate([eye.ravel(), np.zeros(64, np.float32), eye.ravel(), np.zeros(64, np.float32)])
    obs = np.resize(XS, (B, 64)).astype(np.float32)
    tgt = np.zeros((B, 64), np.float32)
    code = mlp.code(hidden)
    one, bc = be.zeros(1), be.zeros(B * 64)
    be.eval_mlp_center(dims, dev(be, theta), dev(be, obs), dev(be, tgt), one, bc, B, B * 64, precision=mode, act=code)
    got = bc.cpu().numpy().reshape(B, 64)
    assert np.isfinite(got).all() and np.isfinite(float(one))
    if mode == "fp32":
        y = torch.from_numpy(obs).cuda()
        want = {"elu": lambda: F.elu(y), "leaky_relu": lambda: F.leaky_relu(y),
                "silu": lambda: y / (1.0 + torch.exp(-y))}[hidden]().cpu().numpy()
        np.testing.assert_array_equal(got, want)                  # the device's IEEE functions, bit for bit
        assert got[0, 1] == (-1.0 if hidden == "elu" else 0.0 if hidden == "silu" else -1.0)
    else:
        want = mlp.FORWARD[mode](theta, dims, obs, hidden)
        np.testing.assert_allclose(got, want, rtol=1e-6, atol=0)
        if mode == "f16" and hidden != "leaky_relu":
            assert got.min() >= -1.0 and got.max() == 65504.0     # only the positive side saturates


# ------------------------------------------------------------------ north-star shape
@pytest.mark.parametrize("hidden", mlp.NEW_KINDS)
def test_north_star_fp32_and_f16_vs_cpu_oracle(be, hidden):
    """P = 4096, n = 1,001,760, B = 256: 512 members (the + and - of 256 pairs) of the fp32 and f16
    device evaluate against the CPU oracle's fp32 forward (max-norm relative)."""
    dims = [128, 512, 512, 512, 512, 288]
    code = mlp.code(hidden)
    n, P, pairs, sigma = orc.mlp_param_count(dims), 4096, 2048, 0.02
    torch.manual_seed(0)
    mods = []
    for i in range(len(dims) - 1):
        l = torch.nn.Linear(dims[i], dims[i + 1])
        mods += [l.weight.detach().reshape(-1), l.bias.detach()]
    theta = torch.cat(mods).contiguous()
    g = torch.Generator().manual_seed(1234)
    obs, tgt = torch.randn(256, 128, generator=g), torch.randn(256, 288, generator=g)
    table = be.alloc(1 << 26)
    be.fill_noise_table(table, 42)
    offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(42, None, 0, 0, pairs, table.numel(), n, offs, order)
    tb16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, tb16) == 0
    assert be.eval_supports_f16(dims, 256, act=code)
    th_d, obs_d, tgt_d = theta.to(be.device), obs.to(be.device), tgt.to(be.device)
    res = {}
    for mode in ("fp32", "f16"):
        r = be.zeros(P)
        be.eval_mlp(dims, th_d, table, offs, order, pairs, sigma, obs_d, tgt_d, r[:pairs], r[pairs:], precision=mode,
                    act=code, **({"table16": tb16} if mode == "f16" else {}))
        res[mode] = r.cpu().numpy()
    tab_h, offs_h, th_h = table.cpu().numpy(), offs.cpu().numpy(), theta.numpy()
    sel = np.arange(0, pairs, pairs // 256)
    want_p, want_m = [], []
    for c in range(0, sel.size, 32):
        pop, _ = orc.sample_population(th_h, tab_h, offs_h[sel[c: c + 32]], sigma)
        w, _ = mlp.evaluate_population(pop, dims, obs.numpy(), tgt.numpy(), mlp.code(hidden))
        want_p.append(w[:len(w) // 2])
        want_m.append(w[len(w) // 2:])
    want = np.concatenate(want_p + want_m)
    idx = np.concatenate([sel, pairs + sel])
    report = {"hidden": hidden, "members_compared": int(idx.size),
              "fp32_max_rel_err": rel_err(res["fp32"][idx], want), "f16_max_rel_err": rel_err(res["f16"][idx], want)}
    print("NORTH_STAR_ACT_EXT " + json.dumps(report))
    assert report["fp32_max_rel_err"] < 2e-6
    assert report["f16_max_rel_err"] < 1e-5


# ------------------------------------------------------------------ public API vs the reference goldens
def _set_theta(module, flat):
    torch.nn.utils.vector_to_parameters(torch.from_numpy(flat.copy()).to(next(module.parameters()).device),
                                        module.parameters())


@pytest.mark.parametrize("fixture,hidden,loss", [("es_elu_cartpole_p64.npz", "elu", "mse"),
                                                 ("es_leaky_xent_p64.npz", "leaky_relu", "xent")])
def test_es_fused_vs_reference_golden(fixture, hidden, loss):
    g = load_golden(fixture)
    dims = [int(d) for d in g["dims"]]
    rec = []

    class R(E.ES):
        def log(self):
            rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                            best=self.best_reward))
    akw = dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]))
    if loss == "xent":
        akw["loss"] = "cross_entropy"
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.1,
           policy_kwargs={"dims": dims, "hidden": hidden}, agent_kwargs=akw, optimizer_kwargs={"lr": 0.01},
           noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]))
    assert es._fused and es._be.name == "cuda" and es._act_code() == mlp.code(hidden, "identity", loss)
    es._table.copy_(torch.from_numpy(g["table"]))
    _set_theta(es.policy, g["theta0"])
    es.train(n_steps=3)
    for gen in range(3):
        assert rel_err(rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-4
        assert abs(rec[gen]["episode"] - float(g["episode_reward"][gen])) < 1e-4
    assert rec[2]["best"] == pytest.approx(float(g["best_reward"][2]), abs=1e-4)
    theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().cpu().numpy()
    assert rel_err(theta, g["theta_after"][2]) < 5e-3


def test_nsr_fused_silu_vs_reference_golden():
    g = load_golden("nsr_silu_bipedal_p32.npz")
    dims = [int(d) for d in g["dims"]]
    rec = []

    class R(E.NSR_ES):
        def log(self):
            rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward, idx=self.idx))
    np.random.seed(123)
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=32, sigma=0.02,
           policy_kwargs={"dims": dims, "hidden": "silu", "output": "tanh"},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]),
                             bc_obs=64, bc_dim=256),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]))
    assert es._fused and es._spec.act == mlp.code("silu", "tanh")
    es._table.copy_(torch.from_numpy(g["table"]))
    for i, (p, _) in enumerate(es.meta_population):
        _set_theta(p, g["meta_theta0"][i])
    es._archive = [a.copy() for a in g["archive0"]]
    np.random.seed(123)
    es.train(n_steps=len(g["grad"]))
    for gen in range(len(g["grad"])):
        assert rec[gen]["idx"] == int(g["idx"][gen])
        assert rel_err(rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-4
        assert rel_err(rec[gen]["returns"][:, 1], g["returns"][gen][:, 1]) < 1e-4
        assert abs(rec[gen]["episode"] - float(g["episode_reward"][gen])) < 1e-4
    np.testing.assert_allclose(np.stack(es._archive), g["archive_final"], rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("hidden", mlp.NEW_KINDS)
def test_auto_picks_f16_and_trains_fused(hidden):
    dims = [128, 256, 64]
    g = torch.Generator().manual_seed(8)
    obs, tgt = torch.randn(256, 128, generator=g), torch.rand(256, 64, generator=g) * 1.8 - 0.9
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.02,
              policy_kwargs={"dims": dims, "hidden": hidden}, agent_kwargs=dict(obs=obs, target=tgt),
              optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 18)
    es.log = lambda: None
    assert es._fused and es._precision == "f16"
    es.train(n_steps=3)
    with torch.no_grad():
        want = float(-((es.policy(obs.cuda()) - tgt.cuda()) ** 2).mean())
    assert abs(es.episode_reward - want) < 1e-4 * abs(want)
