"""Cross-entropy objective without a GPU: ``DeviceAgent(loss="cross_entropy")``, the loss bit of
``estk_mlp_desc.activation`` through the library's shape query, the fused / hooks decision, and ES /
NSR-ES through the oracle stand-in (tests/_xent_oracle.py) against the reference-generated goldens."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden, rel_err
import _xent_oracle as xo
from _xent_oracle import MLP, XentOracleBackend
import estorch_b200 as E
from estorch_b200 import _capi


# ------------------------------------------------------------------ the agent
def _policy_and_batch(B=32, C_=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    pol = MLP([6, 16, C_])
    obs = torch.randn(B, 6, generator=g)
    labels = torch.randint(0, C_, (B,), generator=g)
    return pol, obs, labels, g


def test_rollout_matches_torch_cross_entropy_with_hard_targets():
    pol, obs, labels, _ = _policy_and_batch()
    onehot = F.one_hot(labels, 5).to(torch.float32)
    r = E.DeviceAgent(obs, onehot, loss="cross_entropy").rollout(pol)
    with torch.no_grad():
        want = float(F.cross_entropy(pol(obs), labels))
    assert abs(r + want) <= 1e-6 * abs(want)


def test_rollout_matches_torch_cross_entropy_with_probability_targets():
    pol, obs, _, g = _policy_and_batch(seed=1)
    probs = torch.softmax(torch.randn(32, 5, generator=g), 1)
    r = E.DeviceAgent(obs, probs, loss="cross_entropy").rollout(pol)
    with torch.no_grad():
        want = float(F.cross_entropy(pol(obs), probs))
        logits = pol(obs).numpy()
    assert abs(r + want) <= 1e-6 * abs(want)
    assert abs(r - float(xo.xent_return(logits, probs.numpy()))) <= 1e-6 * abs(want)


def test_rollout_with_behaviour_characteristic_returns_the_logits():
    pol, obs, labels, _ = _policy_and_batch(seed=2)
    r, bc = E.DeviceAgent(obs, F.one_hot(labels, 5).float(), bc_obs=4, bc_dim=18, loss="cross_entropy").rollout(pol)
    with torch.no_grad():
        np.testing.assert_array_equal(bc, pol(obs)[:4].flatten()[:18].numpy())
    assert isinstance(r, float)


def test_default_loss_is_the_squared_error():
    pol, obs, _, g = _policy_and_batch(seed=3)
    tgt = torch.randn(32, 5, generator=g)
    a = E.DeviceAgent(obs, tgt)
    assert a.loss == "mse"
    with torch.no_grad():
        assert a.rollout(pol) == float(-((pol(obs) - tgt) ** 2).mean())


@pytest.mark.parametrize("target,loss", [
    (torch.ones(4, 3), "xent"),
    (torch.ones(4, 3), "MSE"),
    (-torch.ones(4, 3), "cross_entropy"),
    (torch.tensor([[0.5, float("nan"), 0.5]] * 4), "cross_entropy"),
    (torch.tensor([[0.0, float("inf"), 0.0]] * 4), "cross_entropy"),
    (torch.ones(4, 3, dtype=torch.int64), "cross_entropy"),
])
def test_invalid_loss_or_targets_raise(target, loss):
    with pytest.raises(ValueError):
        E.DeviceAgent(torch.randn(4, 2), target, loss=loss)


def test_loss_is_keyword_only():
    with pytest.raises(TypeError):
        E.DeviceAgent(torch.randn(4, 2), torch.ones(4, 3), 0, 0, "cross_entropy")


# ------------------------------------------------------------------ the loss bit in the C ABI
def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


def _supported(lib, dims, act, precision, B=256):
    from estorch_b200.backend import mlp_desc
    d = mlp_desc(dims, act)
    return lib.estk_eval_mlp_supported(C.byref(d), precision, B)


def test_supported_query_accepts_xent_under_the_shape_rule_and_refuses_other_loss_codes():
    lib = _lib()
    assert _capi.ESTK_LOSS_XENT == xo.LOSS_XENT == 0x10000
    north = [128, 512, 512, 512, 512, 256]
    for prec in (_capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S):
        for code in (0x10000, 0x10001):
            assert _supported(lib, north, code, prec) == 1
            assert _supported(lib, [64, 64, 32], code, prec) == 1
            assert _supported(lib, [784, 100, 10], code, prec) == 0          # the shape rule is unchanged
            assert _supported(lib, north, code, prec, B=100) == 0
        for code in (0x10101, 0x20000, 0x10200, 0x10100, 0x1000000, 0x10002):
            assert _supported(lib, north, code, prec) == 0, hex(code)
        for code in (0, 1, 0x100, 0x101):                                     # the existing codes
            assert _supported(lib, north, code, prec) == 1
    assert _supported(lib, north, 0x10000, _capi.ESTK_PREC_FP32) == 0         # not a tensor-core precision


# ------------------------------------------------------------------ fused or hooks
class AtariPolicy(torch.nn.Module):
    """The conv + VirtualBatchNorm policy of the reference's examples/atari.py:14-37."""
    def __init__(self, n_actions, xref):
        super().__init__()
        self.xref = xref
        self.conv1 = torch.nn.Conv2d(4, 16, 8, 4)
        self.bn1 = E.VirtualBatchNorm(16)
        self.conv2 = torch.nn.Conv2d(16, 32, 4, 2)
        self.bn2 = E.VirtualBatchNorm(32)
        self.fc1 = torch.nn.Linear(2592, 256)
        self.fc2 = torch.nn.Linear(256, n_actions)

    def forward(self, x):
        xref = F.relu(self.bn1(self.conv1(self.xref.to(x.device))))
        xref = F.relu(self.bn2(self.conv2(xref)))
        x = F.relu(self.bn1(self.conv1(x)))
        x = F.relu(self.bn2(self.conv2(x)))
        return self.fc2(F.relu(self.fc1(x.view(-1, 2592))))


def _es(hidden, output, loss, tensor_core=False, dims=None, B=None):
    dims = dims or ([64, 64, 32] if tensor_core else [4, 16, 3])
    B = B or (256 if tensor_core else 8)
    rng = np.random.RandomState(3)
    obs = torch.from_numpy(rng.standard_normal((B, dims[0])).astype(np.float32))
    tgt = torch.from_numpy(rng.dirichlet(np.ones(dims[-1]), B).astype(np.float32))
    be = XentOracleBackend(tensor_core=tensor_core)
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
              policy_kwargs={"dims": dims, "hidden": hidden, "output": output},
              agent_kwargs=dict(obs=obs, target=tgt, loss=loss), optimizer_kwargs={"lr": 0.01},
              noise_table_size=1 << 16, _backend=be)
    es.log = lambda: None
    return es, be, obs, tgt


@pytest.mark.parametrize("hidden,output,fused", [("relu", "identity", True), ("tanh", "identity", True),
                                                 ("relu", "tanh", False), ("tanh", "tanh", False)])
def test_decide_fused_for_cross_entropy_mlps(hidden, output, fused):
    es, _, _, _ = _es(hidden, output, "cross_entropy")
    assert es._fused == fused
    assert _es(hidden, output, "mse")[0]._fused                               # the squared error: always fused


def test_cross_entropy_conv_policy_runs_in_hooks_mode():
    g = torch.Generator().manual_seed(5)
    xref = torch.rand(2, 4, 84, 84, generator=g)
    obs = torch.rand(2, 4, 84, 84, generator=g)
    kw = dict(population_size=4, sigma=0.02, policy_kwargs=dict(n_actions=4, xref=xref),
              optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 20)
    xent = E.ES(AtariPolicy, E.DeviceAgent, torch.optim.Adam, agent_kwargs=dict(
        obs=obs, target=F.one_hot(torch.tensor([0, 3]), 4).float(), loss="cross_entropy"),
        _backend=XentOracleBackend(), **kw)
    assert xent._is_conv and not xent._fused
    xent.agent.loss = "mse"                     # the same policy and batch with the squared error is fused
    assert xent._decide_fused(torch.optim.Adam)


@pytest.mark.parametrize("hidden", ["relu", "tanh"])
@pytest.mark.parametrize("tensor_core", [False, True])
def test_the_loss_bit_reaches_every_evaluate_and_auto_picks_f16(hidden, tensor_core):
    es, be, obs, tgt = _es(hidden, "identity", "cross_entropy", tensor_core)
    code = xo.LOSS_XENT | (1 if hidden == "tanh" else 0)
    assert es._fused and es._act_code() == code
    assert es._precision == ("f16" if tensor_core else "fp32")
    es.train(n_steps=3)
    assert be.acts == {code}
    with torch.no_grad():
        want = float(F.cross_entropy(es.policy(obs), tgt))
    assert abs(es.episode_reward + want) < (1e-5 if not tensor_core else 1e-4) * abs(want)


# ------------------------------------------------------------------ against the reference goldens
class _Rec:
    def log(self):
        self.rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                             best=self.best_reward, idx=getattr(self, "idx", None),
                             archive=len(getattr(self, "_archive", []))))


class HostXentAgent:
    """A plain reference-protocol agent with the same rollout: forces hooks mode."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        self.inner = E.DeviceAgent(obs, target, bc_obs, bc_dim, loss="cross_entropy")

    def rollout(self, policy):
        return self.inner.rollout(policy)


def _load_theta(module, flat):
    torch.nn.utils.vector_to_parameters(torch.from_numpy(flat.copy()), module.parameters())


@pytest.mark.parametrize("mode", ["fused", "hooks"])
def test_es_cross_entropy_matches_reference_golden(mode):
    g = load_golden("es_xent_p64.npz")
    dims = [int(d) for d in g["dims"]]

    class R(_Rec, E.ES):
        pass
    agent = E.DeviceAgent if mode == "fused" else HostXentAgent
    akw = dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]))
    if mode == "fused":
        akw["loss"] = "cross_entropy"
    es = R(MLP, agent, torch.optim.Adam, population_size=64, sigma=0.1, policy_kwargs={"dims": dims},
           agent_kwargs=akw, optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]),
           noise_seed=int(g["noise_seed"]), _backend=XentOracleBackend())
    es.rec = []
    assert es._fused == (mode == "fused")
    es._table.copy_(torch.from_numpy(g["table"]))
    _load_theta(es.policy, g["theta0"])
    if mode == "fused":
        es._slots[0].ensure_flat()
    es.train(n_steps=3)
    for gen in range(3):
        assert rel_err(es.rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-5
        assert abs(es.rec[gen]["episode"] - float(g["episode_reward"][gen])) < 2e-5
        assert abs(es.rec[gen]["best"] - float(g["best_reward"][gen])) < 2e-5
    theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().numpy()
    assert rel_err(theta, g["theta_after"][2]) < 2e-4
    bp = es.best_policy_dict
    assert rel_err(np.concatenate([v.reshape(-1).numpy() for v in bp.values()]), g["best_theta"]) < 2e-4


@pytest.mark.parametrize("mode", ["fused", "hooks"])
def test_nsr_cross_entropy_matches_reference_golden(mode):
    g = load_golden("nsr_xent_p32.npz")
    dims = [int(d) for d in g["dims"]]

    class R(_Rec, E.NSR_ES):
        pass
    agent = E.DeviceAgent if mode == "fused" else HostXentAgent
    akw = dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]), bc_obs=64, bc_dim=256)
    if mode == "fused":
        akw["loss"] = "cross_entropy"
    np.random.seed(123)
    es = R(MLP, agent, torch.optim.Adam, population_size=32, sigma=0.02, policy_kwargs={"dims": dims},
           agent_kwargs=akw, optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]),
           noise_seed=int(g["noise_seed"]), _backend=XentOracleBackend())
    es.rec = []
    assert es._fused == (mode == "fused")
    es._table.copy_(torch.from_numpy(g["table"]))
    for i, (p, _) in enumerate(es.meta_population):
        _load_theta(p, g["meta_theta0"][i])
        if mode == "fused":
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
    final = np.stack([torch.nn.utils.parameters_to_vector(p.parameters()).detach().numpy()
                      for p, _ in es.meta_population])
    assert rel_err(final, g["meta_theta_final"]) < 5e-3
    np.testing.assert_allclose(np.stack(es._archive), g["archive_final"], rtol=1e-3, atol=1e-4)


def test_oracle_cross_entropy_reproduces_the_golden_returns():
    from oracle import es_oracle as orc
    g = load_golden("es_xent_p64.npz")
    dims = [int(d) for d in g["dims"]]
    pop, _ = orc.sample_population(g["theta_before"][0], g["table"], g["offsets"][0], np.float32(g["sigma"]))
    rets, _ = xo.evaluate_population(pop, dims, g["obs"], g["target"])
    assert rel_err(rets, g["returns"][0][:, 0]) < 2e-6
    assert np.all(g["returns"][0][:, 0] < 0)
