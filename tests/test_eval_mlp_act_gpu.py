"""Tanh MLP policies on the H100: every MLP evaluate entry point with the four activation codes of
include/estk.h (hidden ReLU / Tanh x output identity / Tanh), against the reference-generated Tanh
goldens and the activation-aware oracle (tests/_act_oracle.py); the north-star shape in fp32 and
f16; and the public API (ES / NSR-ES fused runs, CUDA-graph replay, an f16 fused generation)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import es_oracle as orc
import _act_oracle as act
from _act_oracle import ALL_ACTS, ActOracleBackend, kinds
from test_activations_cpu import ActMLP
import estorch_b200 as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def _set_theta(module, flat):
    with torch.no_grad():
        idx = 0
        for p in module.parameters():
            p.data.copy_(torch.from_numpy(flat[idx: idx + p.numel()]).view(p.shape))
            idx += p.numel()


def dev(be, a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(be.device)


def _eval(be, dims, theta, table, offs, sigma, obs, tgt, act_code, bc_obs=0, bc_dim=0, precision="fp32",
          centre=False, **kw):
    pairs = len(offs)
    ret = be.zeros(2 * pairs)
    bcp = be.zeros(pairs, bc_dim) if bc_dim else None
    bcm = be.zeros(pairs, bc_dim) if bc_dim else None
    c_out = be.zeros(1) if centre else None
    order = dev(be, np.argsort(offs, kind="stable").astype(np.int32))
    be.eval_mlp(dims, dev(be, theta), dev(be, table), dev(be, offs), order, pairs, sigma, dev(be, obs), dev(be, tgt),
                ret[:pairs], ret[pairs:], bcp, bcm, bc_obs, bc_dim, precision=precision, centre_out=c_out,
                act=act_code, **kw)
    torch.cuda.synchronize()
    bcs = None if not bc_dim else np.concatenate([bcp.cpu().numpy(), bcm.cpu().numpy()])
    return ret.cpu().numpy(), bcs, (None if c_out is None else float(c_out))


# ------------------------------------------------------------------ fp32 CUDA-core path
def test_fp32_tanh_matches_reference_goldens(be):
    g = load_golden("es_tanh_cartpole_p64.npz")
    dims = [int(d) for d in g["dims"]]
    for gen in range(len(g["grad"])):
        ret, _, _ = _eval(be, dims, g["theta_before"][gen], g["table"], g["offsets"][gen], float(g["sigma"]),
                          g["obs"], g["target"], act.ACT_TANH)
        assert rel_err(ret, g["returns"][gen][:, 0]) < 2e-6
    g = load_golden("nsr_tanh_bipedal_p32.npz")
    dims, code = [int(d) for d in g["dims"]], act.ACT_TANH | act.ACT_OUT_TANH
    theta, offs = g["theta_before"][0], g["offsets"][0]
    ret, bcs, _ = _eval(be, dims, theta, g["table"], offs, float(g["sigma"]), g["obs"], g["target"], code,
                        bc_obs=64, bc_dim=256)
    assert rel_err(ret, g["returns"][0][:, 0]) < 2e-6
    pop, _ = orc.sample_population(theta, g["table"], offs, float(g["sigma"]))
    _, want_bc = act.evaluate_population(pop, dims, g["obs"], g["target"], 64, 256, "tanh", "tanh")
    assert rel_err(bcs, want_bc) < 2e-6
    # centre entry point: the archive's first entry is the BC of meta_theta0[0]
    one, bc1 = be.zeros(1), be.zeros(256)
    be.eval_mlp_center(dims, dev(be, g["meta_theta0"][0]), dev(be, g["obs"]), dev(be, g["target"]), one, bc1, 64, 256,
                       act=code)
    assert rel_err(bc1.cpu().numpy(), g["archive0"][0]) < 2e-6


@pytest.mark.parametrize("act_code", ALL_ACTS)
@pytest.mark.parametrize("dims,B,pairs", [([128, 512, 512, 288], 48, 4), ([17, 33, 5], 100, 6), ([4, 2], 1, 3),
                                          ([9, 130, 70, 70, 3], 256, 3)])
def test_fp32_shapes_vs_oracle(be, dims, B, pairs, act_code):
    hidden, output = kinds(act_code)
    rng = np.random.RandomState(1)
    n = orc.mlp_param_count(dims)
    table_len = max(1 << 14, (n + 31) // 32 * 32 + 4096)
    table = rng.standard_normal(table_len).astype(np.float32)
    theta = (rng.standard_normal(n) * 0.1).astype(np.float32)
    obs = rng.standard_normal((B, dims[0])).astype(np.float32)
    tgt = rng.standard_normal((B, dims[-1])).astype(np.float32)
    offs = orc.noise_offsets(5, 0, 0, pairs, table_len, n)
    ret, _, _ = _eval(be, dims, theta, table, offs, 0.02, obs, tgt, act_code)
    pop, _ = orc.sample_population(theta, table, offs, 0.02)
    want, _ = act.evaluate_population(pop, dims, obs, tgt, hidden=hidden, output=output)
    assert rel_err(ret, want) < 5e-6
    one = be.zeros(1)
    be.eval_mlp_center(dims, dev(be, theta), dev(be, obs), dev(be, tgt), one, act=act_code)
    w = float(orc.synthetic_return(act.mlp_forward(theta, dims, obs, hidden, output), tgt))
    assert abs(float(one) - w) < 5e-6 * abs(w) + 1e-7


# ------------------------------------------------------------------ tensor-core paths
def _tc_problem(dims, B, pairs, seed=23):
    rng = np.random.RandomState(seed)
    n = orc.mlp_param_count(dims)
    table_len = (n + 31) // 32 * 32 + (1 << 14)
    table = orc.round_f16(rng.standard_normal(table_len).astype(np.float32))   # fp16-exact, like the engine's
    theta = np.concatenate([np.concatenate([(rng.uniform(-1, 1, dims[i] * dims[i + 1]) / np.sqrt(dims[i])),
                                            rng.uniform(-1, 1, dims[i + 1]) / np.sqrt(dims[i])])
                            for i in range(len(dims) - 1)]).astype(np.float32)
    obs = rng.standard_normal((B, dims[0])).astype(np.float32)
    tgt = rng.standard_normal((B, dims[-1])).astype(np.float32)
    offs = orc.noise_offsets(11, 0, 0, pairs, table_len, n)
    return n, table, theta, obs, tgt, offs


# per mode: (vs its emulation, vs the exact fp32 forward, BC vs emulation) -- the ReLU tests' bars
TC_TOL = {"f16": (1e-5, 3e-5, 2e-3), "bf16": (5e-4, 2e-2, 5e-3), "bf16s": (5e-4, 3e-2, 5e-3)}


@pytest.mark.parametrize("act_code", ALL_ACTS)
@pytest.mark.parametrize("mode", ["f16", "bf16", "bf16s"])
@pytest.mark.parametrize("dims,B,pairs,bc", [([64, 256, 64], 512, 4, 256), ([128, 512, 512, 288], 256, 3, 0)])
def test_tensor_core_modes_vs_emulation_and_fp32(be, dims, B, pairs, bc, mode, act_code):
    hidden, output = kinds(act_code)
    n, table, theta, obs, tgt, offs = _tc_problem(dims, B, pairs)
    assert be.eval_supports_f16(dims, B, act=act_code) and be.eval_supports_bf16(dims, B, act=act_code)
    th, tb = dev(be, theta), dev(be, table)
    kw = {}
    if mode == "f16":
        kw["table16"] = be.alloc(table.size, dtype=torch.float16)
        assert be.shadow_f16(tb, kw["table16"]) == 0
    elif mode == "bf16s":
        kw["theta16"], kw["table16"] = be.alloc(n, dtype=torch.bfloat16), be.alloc(table.size, dtype=torch.bfloat16)
        be.shadow_bf16(th, kw["theta16"])
        be.shadow_bf16(tb, kw["table16"])
    got, got_bc, centre = _eval(be, dims, theta, table, offs, 0.02, obs, tgt, act_code, 64 if bc else 0, bc,
                                precision=mode, centre=True, **kw)
    emu_be = ActOracleBackend(tensor_core=True)
    rows = emu_be._rows(torch.from_numpy(theta), torch.from_numpy(table), torch.from_numpy(offs), 0.02, dims, mode)
    emu, emu_bc = act.evaluate_population(rows, dims, obs, tgt, 64 if bc else 0, bc, hidden, output, precision=mode)
    pop, _ = orc.sample_population(theta, table, offs, 0.02)
    exact, exact_bc = act.evaluate_population(pop, dims, obs, tgt, 64 if bc else 0, bc, hidden, output)
    t_emu, t_exact, t_bc = TC_TOL[mode]
    print(f"{mode} act={act_code:#x} {dims}: vs emulation {rel_err(got, emu):.2e}, vs fp32 {rel_err(got, exact):.2e}")
    assert rel_err(got, emu) < t_emu
    assert rel_err(got, exact) < t_exact
    if bc:
        assert rel_err(got_bc, emu_bc) < t_bc
        if mode == "f16":
            assert rel_err(got_bc, exact_bc) < 2e-3
    # the folded centre task and the *_center_* entry point evaluate theta itself
    one = be.zeros(1)
    be.eval_mlp_center(dims, th, dev(be, obs), dev(be, tgt), one, precision=mode, act=act_code,
                       **({"theta16": kw["theta16"]} if mode == "bf16s" else {}))
    ct = torch.zeros(1)
    emu_be.eval_mlp_center(dims, torch.from_numpy(theta), torch.from_numpy(obs), torch.from_numpy(tgt), ct,
                           precision=mode, act=act_code)
    assert abs(float(one) - float(ct)) < t_emu * abs(float(ct))
    assert centre == float(one)                          # same task, same arithmetic, same bits


# ------------------------------------------------------------------ ABI: activation codes
def test_invalid_activation_codes_are_refused(be):
    from estorch_b200 import _capi
    from estorch_b200.backend import mlp_desc
    lib = _capi.load()
    dims, B = [64, 64, 32], 256
    for code in ALL_ACTS:
        d = mlp_desc(dims, code)
        assert lib.estk_eval_mlp_f16_supported(C.byref(d), B) == 1
        assert lib.estk_eval_mlp_bf16_supported(C.byref(d), B) == 1
    n, table, theta, obs, tgt, offs = _tc_problem(dims, B, 2)
    for code in (2, 0x200, 0x101 | 0x10000, -1, 0xff, 1 << 9):
        d = mlp_desc(dims, code)
        assert lib.estk_eval_mlp_f16_supported(C.byref(d), B) == 0
        assert lib.estk_eval_mlp_bf16_supported(C.byref(d), B) == 0
        ret, one = be.zeros(4), be.zeros(1)
        args = (dev(be, theta), dev(be, table), dev(be, offs), None, 2, 0.02, dev(be, obs), dev(be, tgt),
                ret[:2], ret[2:])
        with pytest.raises(RuntimeError, match=r"estk_status -1\)"):
            be.eval_mlp(dims, *args, act=code)
        with pytest.raises(RuntimeError, match=r"estk_status -1\)"):
            be.eval_mlp_center(dims, dev(be, theta), dev(be, obs), dev(be, tgt), one, act=code)
        with pytest.raises(RuntimeError, match="not supported"):
            be.eval_mlp(dims, *args, act=code, precision="bf16")
    torch.cuda.synchronize()


# ------------------------------------------------------------------ north-star shape
@pytest.mark.parametrize("output", ["identity", "tanh"])
def test_north_star_tanh_fp32_and_f16_vs_cpu_oracle(be, output):
    """P = 4096, n = 1,001,760, B = 256, Tanh hidden: 512 members (the + and - of 256 pairs) of the
    fp32 and f16 device evaluate against the CPU oracle's fp32 forward (max-norm relative)."""
    dims = [128, 512, 512, 512, 512, 288]
    code = act.code("tanh", output)
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
    sel = np.arange(0, pairs, pairs // 256)                       # 256 pairs spread over the population
    want_p, want_m = [], []
    for c in range(0, sel.size, 32):                              # 64 rows (256 MB) at a time
        pop, _ = orc.sample_population(th_h, tab_h, offs_h[sel[c: c + 32]], sigma)
        w, _ = act.evaluate_population(pop, dims, obs.numpy(), tgt.numpy(), hidden="tanh", output=output)
        want_p.append(w[:len(w) // 2])
        want_m.append(w[len(w) // 2:])
    want = np.concatenate(want_p + want_m)
    idx = np.concatenate([sel, pairs + sel])
    report = {"hidden": "tanh", "output": output, "members_compared": int(idx.size),
              "fp32_max_rel_err": rel_err(res["fp32"][idx], want), "f16_max_rel_err": rel_err(res["f16"][idx], want)}
    print("NORTH_STAR_TANH " + json.dumps(report))
    assert report["fp32_max_rel_err"] < 2e-6
    assert report["f16_max_rel_err"] < 1e-5


# ------------------------------------------------------------------ public API
def test_es_fused_tanh_vs_reference_golden():
    g = load_golden("es_tanh_cartpole_p64.npz")
    dims = [int(d) for d in g["dims"]]
    rec = []

    class R(E.ES):
        def log(self):
            rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                            best=self.best_reward, grad=self._grad.cpu().numpy().copy(),
                            theta=self._slots[0].theta.cpu().numpy().copy()))
    es = R(ActMLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.1,
           policy_kwargs={"dims": dims, "hidden": "tanh"},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"])),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]))
    assert es._fused and es._be.name == "cuda" and es._spec.act == act.ACT_TANH
    es._table.copy_(torch.from_numpy(g["table"]))
    _set_theta(es.policy, g["theta0"])
    es.train(n_steps=3)
    theta, m, v = g["theta0"].copy(), np.zeros(es.n_parameters, np.float32), np.zeros(es.n_parameters, np.float32)
    for gen in range(3):
        r = rec[gen]
        pop, eps = orc.sample_population(theta, g["table"], g["offsets"][gen], 0.1)
        want, _ = act.evaluate_population(pop, dims, g["obs"], g["target"], hidden="tanh")
        assert rel_err(r["returns"][:, 0], want) < 5e-6
        assert rel_err(r["grad"], orc.calculate_grad(r["returns"][:, 0], eps, 0.1)) < 1e-5
        th, m, v = orc.adam_step(theta, m, v, orc.negate_clamp(r["grad"]), gen + 1)
        assert rel_err(r["theta"], th) < 1e-6
        ep = orc.synthetic_return(act.mlp_forward(th, dims, g["obs"], "tanh"), g["target"])
        assert abs(r["episode"] - float(ep)) < 1e-5
        theta = r["theta"]
        assert rel_err(r["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-4   # the reference's trajectory
    assert rel_err(rec[2]["theta"], g["theta_after"][2]) < 5e-3          # chained Adam steps, sign flips at g~0
    assert rec[2]["best"] == pytest.approx(float(g["best_reward"][2]), abs=1e-4)
    bp = es.best_policy_dict
    assert rel_err(np.concatenate([v_.reshape(-1).cpu().numpy() for v_ in bp.values()]), g["best_theta"]) < 5e-3


def test_nsr_fused_tanh_vs_reference_golden():
    g = load_golden("nsr_tanh_bipedal_p32.npz")
    dims = [int(d) for d in g["dims"]]
    rec = []

    class R(E.NSR_ES):
        def log(self):
            rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward, idx=self.idx))
    np.random.seed(123)
    es = R(ActMLP, E.DeviceAgent, torch.optim.Adam, population_size=32, sigma=0.02,
           policy_kwargs={"dims": dims, "hidden": "tanh", "output": "tanh"},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]),
                             bc_obs=64, bc_dim=256),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]))
    assert es._fused and es._spec.act == act.ACT_TANH | act.ACT_OUT_TANH
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
    final = np.stack([torch.nn.utils.parameters_to_vector(p.parameters()).detach().cpu().numpy()
                      for p, _ in es.meta_population])
    assert rel_err(final, g["meta_theta_final"]) < 5e-3
    np.testing.assert_allclose(np.stack(es._archive), g["archive_final"], rtol=1e-3, atol=1e-4)


def test_graph_replay_equals_eager_tanh(monkeypatch):
    dims = [128, 512, 288]
    g = torch.Generator().manual_seed(2)
    obs, tgt = torch.randn(256, 128, generator=g), torch.rand(256, 288, generator=g) * 1.8 - 0.9
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ESTORCH_B200_GRAPH", mode)
        torch.manual_seed(4)
        es = E.ES(ActMLP, E.DeviceAgent, torch.optim.Adam, population_size=128, sigma=0.02,
                  policy_kwargs={"dims": dims, "hidden": "tanh", "output": "tanh"},
                  agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 22,
                  log_interval=4)
        assert es._precision == "f16" and es._spec.act == act.ACT_TANH | act.ACT_OUT_TANH
        es.log = lambda: None
        es.train(n_steps=13)
        out[mode] = (es._slots[0].theta.clone(), es._slots[0].best_theta.clone(), es.episode_reward, es.best_reward,
                     es.population_returns.copy(), sum(isinstance(v, tuple) for v in es.__dict__.get("_graphs", {}).values()))
    a, b = out["1"], out["0"]
    assert a[5] >= 1 and b[5] == 0
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3]
    np.testing.assert_array_equal(a[4], b[4])


@pytest.mark.parametrize("output", ["identity", "tanh"])
def test_f16_tanh_fused_generation_vs_oracle_emulation(output):
    """One "f16" fused generation of a Tanh policy at a tensor-core shape against the oracle
    stand-in running the same host logic on the f16 emulation."""
    dims = [128, 256, 256, 64]
    g = torch.Generator().manual_seed(8)
    obs, tgt = torch.randn(256, 128, generator=g), torch.rand(256, 64, generator=g) * 1.8 - 0.9
    res, table = {}, None
    for name, backend in (("cuda", None), ("oracle", ActOracleBackend(tensor_core=True))):
        torch.manual_seed(6)
        rec = []

        class R(E.ES):
            def log(self):
                rec.append((self.population_returns.copy(), self.episode_reward,
                            self._slots[0].theta.detach().cpu().numpy().copy()))
        es = R(ActMLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.02,
               policy_kwargs={"dims": dims, "hidden": "tanh", "output": output},
               agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 18,
               eval_precision="f16", _backend=backend)
        assert es._fused and es._precision == "f16"
        if table is None:
            table = es._table.cpu()
        else:                               # the device's Philox table (libm and the device differ in ulps)
            es._table.copy_(table)
        es.train(n_steps=1)
        res[name] = rec[0]
    (r_c, ep_c, th_c), (r_o, ep_o, th_o) = res["cuda"], res["oracle"]
    print(f"f16 tanh/{output} fused generation: returns vs emulation {rel_err(r_c[:, 0], r_o[:, 0]):.2e}")
    assert rel_err(r_c[:, 0], r_o[:, 0]) < 1e-5
    assert abs(ep_c - ep_o) < 1e-5 * abs(ep_o)
    # ranks may swap between returns closer than the kernels' difference; theta moves by at most lr per entry
    assert np.abs(th_c - th_o).max() <= 2 * 0.01 + 1e-6
