"""ELU, SiLU and LeakyReLU MLP policies on the CPU: recognition (estorch_b200.policy_spec), the
activation codes of the C ABI and its support probe, the oracle forwards against the reference-
generated goldens, and the fused generation of ES / NSR-ES through the oracle stand-in
(tests/_act_ext_oracle.py) against the same goldens."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
from torch import nn
import torch.nn.functional as F

from conftest import load_golden, rel_err
from oracle import es_oracle as orc
import _act_ext_oracle as ext
from _act_ext_oracle import MLP, ActExtOracleBackend
import estorch_b200 as E
from estorch_b200 import _capi
from estorch_b200.policy_spec import MLPSpec, mlp_spec_from_module

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ext.NEW_KINDS


# ------------------------------------------------------------------ recognition
@pytest.mark.parametrize("output", ["identity", "tanh"])
@pytest.mark.parametrize("hidden", KINDS)
def test_recognition_of_registered_activations(hidden, output):
    spec = mlp_spec_from_module(MLP([4, 64, 64, 2], hidden, output))
    assert spec == MLPSpec((4, 64, 64, 2), hidden, output)
    assert spec.act == ext.code(hidden, output) == ext.HIDDEN_CODES[hidden] | (256 if output == "tanh" else 0)


@pytest.mark.parametrize("output", ["identity", "tanh"])
@pytest.mark.parametrize("hidden", KINDS)
def test_recognition_of_functional_activations(hidden, output):
    fn = {"elu": F.elu, "silu": F.silu, "leaky_relu": F.leaky_relu}[hidden]

    class Fn(nn.Module):
        def __init__(self):
            super().__init__()
            self.l1, self.l2, self.l3 = nn.Linear(4, 32), nn.Linear(32, 32), nn.Linear(32, 2)

        def forward(self, x):
            y = self.l3(fn(self.l2(fn(self.l1(x)))))
            return torch.tanh(y) if output == "tanh" else y
    assert mlp_spec_from_module(Fn()) == MLPSpec((4, 32, 32, 2), hidden, output)


def test_existing_kinds_are_recognised_as_before():
    assert mlp_spec_from_module(MLP([4, 64, 64, 2], "relu")) == MLPSpec((4, 64, 64, 2))
    assert mlp_spec_from_module(MLP([4, 64, 64, 2], "tanh", "tanh")) == MLPSpec((4, 64, 64, 2), "tanh", "tanh")
    assert mlp_spec_from_module(nn.Linear(3, 2)) == MLPSpec((3, 2))

    class G(nn.Module):                      # functional ReLU is not mistaken for LeakyReLU, nor Tanh for SiLU
        def __init__(self):
            super().__init__()
            self.l1, self.l2 = nn.Linear(4, 32), nn.Linear(32, 2)

        def forward(self, x):
            return self.l2(torch.relu(self.l1(x)))
    assert mlp_spec_from_module(G()) == MLPSpec((4, 32, 2))


@pytest.mark.parametrize("module", [
    nn.Sequential(nn.Linear(4, 64), nn.ELU(alpha=0.5), nn.Linear(64, 2)),
    nn.Sequential(nn.Linear(4, 64), nn.LeakyReLU(0.2), nn.Linear(64, 2)),
    nn.Sequential(nn.Linear(4, 64), nn.ELU(), nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 2)),
    nn.Sequential(nn.Linear(4, 64), nn.SiLU(), nn.Linear(64, 64), nn.LeakyReLU(), nn.Linear(64, 2)),
    nn.Sequential(nn.Linear(4, 64), nn.ELU(), nn.Linear(64, 2), nn.SiLU()),
    nn.Sequential(nn.Linear(4, 64), nn.CELU(), nn.Linear(64, 2)),
])
def test_other_parameters_mixes_and_outputs_are_not_recognised(module):
    assert mlp_spec_from_module(module) is None


def test_functional_leaky_relu_with_another_slope_is_not_recognised():
    class Fn(nn.Module):
        def __init__(self):
            super().__init__()
            self.l1, self.l2 = nn.Linear(4, 32), nn.Linear(32, 2)

        def forward(self, x):
            return self.l2(F.leaky_relu(self.l1(x), 0.2))
    assert mlp_spec_from_module(Fn()) is None


def test_structure_only_recognition_needs_the_probe_for_the_new_kinds():
    assert mlp_spec_from_module(MLP([4, 16, 2], "silu"), probe=False) is None
    assert mlp_spec_from_module(MLP([4, 16, 2], "relu"), probe=False) == MLPSpec((4, 16, 2))


@pytest.mark.parametrize("hidden", KINDS)
def test_recognition_leaves_the_global_rng_stream_as_before(hidden):
    m = MLP([4, 64, 64, 2], hidden, "tanh")
    torch.manual_seed(5)
    mlp_spec_from_module(m)
    a = torch.rand(4)
    torch.manual_seed(5)
    torch.randn(3, 4)
    assert torch.equal(a, torch.rand(4))


# ------------------------------------------------------------------ ABI
def test_header_and_binding_agree_on_the_codes():
    header = open(os.path.join(ROOT, "include", "estk.h")).read()
    for name, want in (("ESTK_ACT_ELU", 3), ("ESTK_ACT_SILU", 4), ("ESTK_ACT_LEAKY_RELU", 5)):
        m = re.search(r"#define\s+%s\s+(\d+)" % name, header)
        assert m and int(m.group(1)) == getattr(_capi, name) == want == ext.HIDDEN_CODES[name[9:].lower()]
    assert not re.search(r"#define\s+ESTK_ACT_\w+\s+2\b", header)              # 2 stays undefined
    assert re.search(r"#define\s+ESTK_VERSION\s+200\b", header)
    from estorch_b200.policy_spec import _HIDDEN_CODES
    assert _HIDDEN_CODES == ext.HIDDEN_CODES


def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


def _supported(lib, dims, code, precision, B):
    from estorch_b200.backend import mlp_desc
    return lib.estk_eval_mlp_supported(C.byref(mlp_desc(dims, code)), precision, B)


REFUSED = [2, 0xff, 0x200, -1, 1 << 24, 0x20000, 0x10200, 6, 0x0102, 0x10002] + \
          [0x10100 | h for h in (0, 1, 3, 4, 5)]


def test_support_probe_takes_the_new_codes_and_refuses_the_rest():
    lib = _lib()
    TC = (_capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S)
    for code in ext.NEW_ACTS:
        for prec in TC:
            assert _supported(lib, [64, 64, 32], code, prec, 256) == 1, (hex(code), prec)
            assert _supported(lib, [64, 64, 32], code, prec, 100) == 0, (hex(code), prec)    # the shape rule
        assert _supported(lib, [320, 64, 32], code, _capi.ESTK_PREC_F16, 256) == 0
        for B in (1, 100, 256, 60000):
            assert _supported(lib, [784, 100, 10], code, _capi.ESTK_PREC_F16_ANY, B) == 1, (hex(code), B)
    for code in REFUSED:
        for prec in TC:
            assert _supported(lib, [64, 64, 32], code, prec, 256) == 0, (hex(code), prec)
        assert _supported(lib, [784, 100, 10], code, _capi.ESTK_PREC_F16_ANY, 100) == 0, hex(code)


# ------------------------------------------------------------------ oracle forward vs the reference goldens
def test_oracle_activations_match_torch():
    y = torch.tensor([-100.0, -30.0, -1.0, -1e-30, -0.0, 0.0, 1e-30, 0.5, 3.0, 100.0])
    yn = y.numpy()
    np.testing.assert_array_equal(ext._leaky_relu(yn), F.leaky_relu(y).numpy())
    np.testing.assert_allclose(ext._elu(yn), F.elu(y).numpy(), rtol=2e-7, atol=0)
    np.testing.assert_allclose(ext._silu(yn), (y / (1 + torch.exp(-y))).numpy(), rtol=2e-7, atol=0)
    assert ext._silu(np.float32([-100.0]))[0] == 0 and ext._elu(np.float32([-100.0]))[0] == -1


def _check_population_golden(g, hidden, output, loss, bc=False):
    dims, sigma = [int(d) for d in g["dims"]], float(g["sigma"])
    bc_obs, bc_dim = (int(g["bc_obs"]), int(g["bc_dim"])) if bc else (0, 0)
    out = []
    for gen in range(len(g["grad"])):
        pop, _ = orc.sample_population(g["theta_before"][gen], g["table"], g["offsets"][gen], sigma)
        rets, bcs = ext.evaluate_population(pop, dims, g["obs"], g["target"], bc_obs, bc_dim, hidden, output,
                                            loss=loss)
        assert rel_err(rets, g["returns"][gen][:, 0]) < 2e-6
        ep = ext.member_return(ext.mlp_forward(g["theta_after"][gen], dims, g["obs"], hidden, output), g["target"],
                               loss)
        assert abs(float(ep) - float(g["episode_reward"][gen])) < 1e-5
        out.append(bcs)
    return out


def test_oracle_elu_forward_matches_reference_golden_es():
    _check_population_golden(load_golden("es_elu_cartpole_p64.npz"), "elu", "identity", "mse")


def test_oracle_leaky_relu_cross_entropy_matches_reference_golden_es():
    _check_population_golden(load_golden("es_leaky_xent_p64.npz"), "leaky_relu", "identity", "xent")


def test_oracle_silu_forward_matches_reference_golden_nsr_bc():
    g = load_golden("nsr_silu_bipedal_p32.npz")
    dims, k = [int(d) for d in g["dims"]], int(g["k"])
    bc_obs, bc_dim = int(g["bc_obs"]), int(g["bc_dim"])
    fwd = lambda th: ext.mlp_forward(th, dims, g["obs"], "silu", "tanh")  # noqa: E731
    archive = [orc.synthetic_bc(fwd(th), bc_obs, bc_dim) for th in g["meta_theta0"]]
    np.testing.assert_allclose(np.stack(archive), g["archive0"], rtol=1e-5, atol=1e-6)
    bcs_all = _check_population_golden(g, "silu", "tanh", "mse", bc=True)
    for gen, bcs in enumerate(bcs_all):
        nov = np.array([orc.novelty(b, np.stack(archive), k) for b in bcs], dtype=np.float32)
        assert rel_err(nov, g["returns"][gen][:, 1]) < 2e-5
        archive.append(orc.synthetic_bc(fwd(g["theta_after"][gen]), bc_obs, bc_dim))
    np.testing.assert_allclose(np.stack(archive), g["archive_final"], rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------ fused generation vs the reference goldens
class _Rec:
    def log(self):
        self.rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                             best=self.best_reward, idx=getattr(self, "idx", None),
                             archive=len(getattr(self, "_archive", []))))


def _load_theta(module, flat):
    torch.nn.utils.vector_to_parameters(torch.from_numpy(flat.copy()), module.parameters())


@pytest.mark.parametrize("fixture,hidden,loss", [("es_elu_cartpole_p64.npz", "elu", "mse"),
                                                 ("es_leaky_xent_p64.npz", "leaky_relu", "xent")])
def test_es_fused_matches_reference_golden(fixture, hidden, loss):
    g = load_golden(fixture)
    dims = [int(d) for d in g["dims"]]

    class R(_Rec, E.ES):
        pass
    akw = dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]))
    if loss == "xent":
        akw["loss"] = "cross_entropy"
    be = ActExtOracleBackend()
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.1,
           policy_kwargs={"dims": dims, "hidden": hidden}, agent_kwargs=akw, optimizer_kwargs={"lr": 0.01},
           noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]), _backend=be)
    es.rec = []
    assert es._fused and es._spec == MLPSpec(tuple(dims), hidden, "identity")
    es._table.copy_(torch.from_numpy(g["table"]))
    _load_theta(es.policy, g["theta0"])
    es._slots[0].ensure_flat()
    es.train(n_steps=3)
    assert be.acts == {ext.code(hidden, "identity", loss)}
    for gen in range(3):
        assert rel_err(es.rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-5
        assert abs(es.rec[gen]["episode"] - float(g["episode_reward"][gen])) < 2e-5
        assert abs(es.rec[gen]["best"] - float(g["best_reward"][gen])) < 2e-5
    theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().numpy()
    assert rel_err(theta, g["theta_after"][2]) < 2e-4
    bp = es.best_policy_dict
    assert rel_err(np.concatenate([v.reshape(-1).numpy() for v in bp.values()]), g["best_theta"]) < 2e-4


def test_nsr_fused_silu_matches_reference_golden():
    g = load_golden("nsr_silu_bipedal_p32.npz")
    dims = [int(d) for d in g["dims"]]

    class R(_Rec, E.NSR_ES):
        pass
    np.random.seed(123)
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=32, sigma=0.02,
           policy_kwargs={"dims": dims, "hidden": "silu", "output": "tanh"},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]), bc_obs=64,
                             bc_dim=256),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]),
           _backend=ActExtOracleBackend())
    es.rec = []
    assert es._fused and es._spec.act == _capi.ESTK_ACT_SILU | _capi.ESTK_ACT_OUT_TANH
    es._table.copy_(torch.from_numpy(g["table"]))
    for i, (p, _) in enumerate(es.meta_population):
        _load_theta(p, g["meta_theta0"][i])
        es._slots[i].push_theta()
    es._archive = [a.copy() for a in g["archive0"]]
    np.random.seed(123)
    es.train(n_steps=len(g["grad"]))
    for gen in range(len(g["grad"])):
        r = es.rec[gen]
        assert r["idx"] == int(g["idx"][gen])
        assert rel_err(r["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-4
        assert rel_err(r["returns"][:, 1], g["returns"][gen][:, 1]) < 1e-4
        assert abs(r["episode"] - float(g["episode_reward"][gen])) < 1e-4
        assert r["archive"] == int(g["archive_len"][gen])
    np.testing.assert_allclose(np.stack(es._archive), g["archive_final"], rtol=1e-3, atol=1e-4)
    assert abs(es.best_reward - float(max(g["episode_reward"]))) < 1e-4


# ------------------------------------------------------------------ fused mode and the codes that reach the kernels
@pytest.mark.parametrize("loss", ["mse", "xent"])
@pytest.mark.parametrize("tensor_core", [False, True])
@pytest.mark.parametrize("hidden", KINDS)
def test_fused_and_the_code_reaches_every_evaluate(hidden, tensor_core, loss):
    dims, B = ([64, 64, 32], 256) if tensor_core else ([4, 16, 2], 8)
    rng = np.random.RandomState(3)
    obs = torch.from_numpy(rng.standard_normal((B, dims[0])).astype(np.float32))
    if loss == "xent":
        tgt = torch.nn.functional.one_hot(torch.from_numpy(rng.randint(0, dims[-1], B)), dims[-1]).float()
    else:
        tgt = torch.from_numpy(rng.uniform(-0.9, 0.9, (B, dims[-1])).astype(np.float32))
    be = ActExtOracleBackend(tensor_core=tensor_core)
    akw = dict(obs=obs, target=tgt)
    if loss == "xent":
        akw["loss"] = "cross_entropy"
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
              policy_kwargs={"dims": dims, "hidden": hidden}, agent_kwargs=akw, optimizer_kwargs={"lr": 0.01},
              noise_table_size=1 << 16, _backend=be)
    es.log = lambda: None
    code = ext.code(hidden, "identity", loss)
    assert es._fused and es._act_code() == code
    assert es._precision == ("f16" if tensor_core else "fp32")       # "auto" picks f16 where the shape allows
    es.train(n_steps=2)
    assert be.acts == {code}


def test_default_elu_is_fused_and_a_nondefault_alpha_stays_in_hooks_mode():
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
              policy_kwargs={"dims": [4, 16, 2], "hidden": "elu"},
              agent_kwargs=dict(obs=torch.randn(8, 4), target=torch.randn(8, 2)), noise_table_size=1 << 12,
              _backend=ActExtOracleBackend())
    assert es._fused

    class Elu05(nn.Module):
        def __init__(self):
            super().__init__()
            self.net = nn.Sequential(nn.Linear(4, 16), nn.ELU(alpha=0.5), nn.Linear(16, 2))

        def forward(self, x):
            return self.net(x)
    es = E.ES(Elu05, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
              agent_kwargs=dict(obs=torch.randn(8, 4), target=torch.randn(8, 2)), noise_table_size=1 << 12,
              _backend=ActExtOracleBackend())
    assert es._spec is None and not es._fused
