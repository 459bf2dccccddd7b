"""Tanh MLP policies on the CPU: recognition (estorch_b200.policy_spec), the activation-aware
oracle forward against the reference-generated Tanh goldens, and the fused generation of the
ES / NSR-ES classes through the oracle stand-in (tests/_oracle_backend.py) against the same goldens."""
import numpy as np
import pytest
import torch
from torch import nn

from conftest import load_golden, rel_err
from oracle import es_oracle as orc
import _mlp_oracle as mlp
from _oracle_backend import OracleBackend
import estorch_b200 as E
from estorch_b200.policy_spec import MLPSpec, mlp_spec_from_module


class ActMLP(nn.Module):
    """Linear -> hidden -> ... -> Linear [-> output], activations as registered modules."""

    def __init__(self, dims, hidden="tanh", output="identity"):
        super().__init__()
        mk = {"relu": nn.ReLU, "tanh": nn.Tanh, "gelu": nn.GELU, "sigmoid": nn.Sigmoid}
        layers = []
        for i in range(len(dims) - 1):
            layers.append(nn.Linear(dims[i], dims[i + 1]))
            if i + 2 < len(dims):
                layers.append(mk[hidden[i] if isinstance(hidden, (list, tuple)) else hidden]())
        if output != "identity":
            layers.append(mk[output]())
        self.net = nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


# ------------------------------------------------------------------ recognition
@pytest.mark.parametrize("hidden,output", [("relu", "identity"), ("tanh", "identity"), ("relu", "tanh"),
                                           ("tanh", "tanh")])
def test_recognition_of_registered_activations(hidden, output):
    spec = mlp_spec_from_module(ActMLP([4, 64, 64, 2], hidden, output))
    assert spec == MLPSpec((4, 64, 64, 2), hidden, output)
    assert spec.act == mlp.code(hidden, output)
    assert spec.n_parameters == 4610


def test_recognition_keeps_relu_spec_and_default_fields():
    assert MLPSpec((3, 2)) == MLPSpec((3, 2), "relu", "identity") and MLPSpec((3, 2)).act == 0
    assert mlp_spec_from_module(nn.Linear(3, 2)) == MLPSpec((3, 2))           # es_tiny_p8's policy
    assert mlp_spec_from_module(nn.Sequential(nn.Linear(3, 2), nn.Tanh())) == MLPSpec((3, 2), "relu", "tanh")


def test_recognition_of_functional_tanh_without_activation_modules():
    class F(nn.Module):
        def __init__(self):
            super().__init__()
            self.l1, self.l2, self.l3 = nn.Linear(4, 32), nn.Linear(32, 32), nn.Linear(32, 2)

        def forward(self, x):
            return torch.tanh(self.l3(torch.tanh(self.l2(torch.tanh(self.l1(x))))))
    assert mlp_spec_from_module(F()) == MLPSpec((4, 32, 32, 2), "tanh", "tanh")

    class G(F):
        def forward(self, x):
            return self.l3(torch.relu(self.l2(torch.relu(self.l1(x)))))
    assert mlp_spec_from_module(G()) == MLPSpec((4, 32, 32, 2))


def test_small_last_layer_tanh_output_is_not_mistaken_for_identity():
    """A last layer initialised at 1e-3 scale makes tanh(y) ~ y to 1e-7 relative on the module's own
    parameters; the probe redraws them, so the output Tanh is still found."""
    m = ActMLP([4, 64, 64, 2], "tanh", "tanh")
    with torch.no_grad():
        m.net[4].weight.mul_(1e-3)
        m.net[4].bias.mul_(1e-3)
    y = m(torch.randn(3, 4))
    assert torch.allclose(torch.tanh(y), y, rtol=1e-4, atol=1e-5)           # indistinguishable as it stands
    assert mlp_spec_from_module(m) == MLPSpec((4, 64, 64, 2), "tanh", "tanh")


@pytest.mark.parametrize("module", [
    ActMLP([4, 64, 64, 2], ["relu", "tanh"]), ActMLP([4, 64, 64, 2], ["tanh", "relu"]),
    ActMLP([4, 64, 64, 2], "gelu"), ActMLP([4, 64, 64, 2], "sigmoid"), ActMLP([4, 64, 64, 2], "relu", "sigmoid")])
def test_unsupported_activations_are_not_recognised(module):
    assert mlp_spec_from_module(module) is None


def test_recognition_leaves_the_global_rng_stream_as_before():
    """ES.__init__ builds the policy after recognising it: the probe must draw from the global
    RNG exactly what it drew before Tanh policies were recognised (one [3, in] normal batch)."""
    m = ActMLP([4, 64, 64, 2], "tanh", "tanh")
    torch.manual_seed(5)
    mlp_spec_from_module(m)
    a = torch.rand(4)
    torch.manual_seed(5)
    torch.randn(3, 4)
    assert torch.equal(a, torch.rand(4))


# ------------------------------------------------------------------ oracle forward vs the reference goldens
def test_oracle_tanh_forward_matches_reference_golden_es():
    g = load_golden("es_tanh_cartpole_p64.npz")
    dims, sigma = [int(d) for d in g["dims"]], float(g["sigma"])
    for gen in range(len(g["grad"])):
        pop, _ = orc.sample_population(g["theta_before"][gen], g["table"], g["offsets"][gen], sigma)
        rets, _ = mlp.evaluate_population(pop, dims, g["obs"], g["target"], mlp.ACT_TANH)
        assert rel_err(rets, g["returns"][gen][:, 0]) < 2e-6
        ep = orc.synthetic_return(orc.mlp_forward(g["theta_after"][gen], dims, g["obs"], "tanh"), g["target"])
        assert abs(float(ep) - float(g["episode_reward"][gen])) < 1e-5
    # the default keywords are the ReLU oracle
    rr, _ = mlp.evaluate_population(pop[:4], dims, g["obs"], g["target"])
    np.testing.assert_array_equal(rr, orc.evaluate_population(pop[:4], dims, g["obs"], g["target"])[0])


def test_oracle_tanh_forward_matches_reference_golden_nsr_bc():
    g = load_golden("nsr_tanh_bipedal_p32.npz")
    dims, sigma, k = [int(d) for d in g["dims"]], float(g["sigma"]), int(g["k"])
    bc_obs, bc_dim = int(g["bc_obs"]), int(g["bc_dim"])
    fwd = lambda th: orc.mlp_forward(th, dims, g["obs"], "tanh", "tanh")  # noqa: E731
    arch0 = np.stack([orc.synthetic_bc(fwd(th), bc_obs, bc_dim) for th in g["meta_theta0"]])
    np.testing.assert_allclose(arch0, g["archive0"], rtol=1e-5, atol=1e-6)
    archive = list(arch0)
    for gen in range(len(g["grad"])):
        pop, _ = orc.sample_population(g["theta_before"][gen], g["table"], g["offsets"][gen], sigma)
        rets, bcs = mlp.evaluate_population(pop, dims, g["obs"], g["target"], mlp.code("tanh", "tanh"), bc_obs=bc_obs,
                                            bc_dim=bc_dim)
        nov = np.array([orc.novelty(b, np.stack(archive), k) for b in bcs], dtype=np.float32)
        assert rel_err(rets, g["returns"][gen][:, 0]) < 2e-6
        assert rel_err(nov, g["returns"][gen][:, 1]) < 2e-5
        out = fwd(g["theta_after"][gen])
        assert abs(float(orc.synthetic_return(out, g["target"])) - float(g["episode_reward"][gen])) < 1e-5
        archive.append(orc.synthetic_bc(out, bc_obs, bc_dim))
    np.testing.assert_allclose(np.stack(archive), g["archive_final"], rtol=1e-4, atol=1e-5)
    assert np.abs(g["archive_final"]).max() <= 1.0                        # BCs are Tanh outputs


# ------------------------------------------------------------------ fused generation vs the reference goldens
class _Rec:
    def log(self):
        self.rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                             best=self.best_reward, idx=getattr(self, "idx", None),
                             archive=len(getattr(self, "_archive", []))))


def _load_theta(module, flat):
    torch.nn.utils.vector_to_parameters(torch.from_numpy(flat.copy()), module.parameters())


def test_es_fused_tanh_matches_reference_golden():
    g = load_golden("es_tanh_cartpole_p64.npz")
    dims = [int(d) for d in g["dims"]]

    class R(_Rec, E.ES):
        pass
    es = R(ActMLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.1,
           policy_kwargs={"dims": dims, "hidden": "tanh"},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"])),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]),
           _backend=OracleBackend())
    es.rec = []
    assert es._fused and es._spec == MLPSpec(tuple(dims), "tanh", "identity")
    es._table.copy_(torch.from_numpy(g["table"]))
    _load_theta(es.policy, g["theta0"])
    es._slots[0].ensure_flat()
    es.train(n_steps=3)
    for gen in range(3):
        assert rel_err(es.rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-5
        assert abs(es.rec[gen]["episode"] - float(g["episode_reward"][gen])) < 2e-5
        assert abs(es.rec[gen]["best"] - float(g["best_reward"][gen])) < 2e-5
    theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().numpy()
    assert rel_err(theta, g["theta_after"][2]) < 2e-4      # 3 chained generations on oracle returns
    grad = es._grad.numpy()                                  # the last generation's estimate
    ok = np.abs(g["grad"][2]) > 1e-4 * np.abs(g["grad"][2]).max()
    assert rel_err(grad[ok], g["grad"][2][ok]) < 1e-3
    bp = es.best_policy_dict
    assert rel_err(np.concatenate([v.reshape(-1).numpy() for v in bp.values()]), g["best_theta"]) < 2e-4


def test_nsr_fused_tanh_matches_reference_golden():
    g = load_golden("nsr_tanh_bipedal_p32.npz")
    dims = [int(d) for d in g["dims"]]

    class R(_Rec, E.NSR_ES):
        pass
    np.random.seed(123)
    es = R(ActMLP, E.DeviceAgent, torch.optim.Adam, population_size=32, sigma=0.02,
           policy_kwargs={"dims": dims, "hidden": "tanh", "output": "tanh"},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]), bc_obs=64,
                             bc_dim=256),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]),
           _backend=OracleBackend())
    es.rec = []
    assert es._fused and es._spec.act == mlp.ACT_TANH | mlp.ACT_OUT_TANH
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
    final = np.stack([torch.nn.utils.parameters_to_vector(p.parameters()).detach().numpy()
                      for p, _ in es.meta_population])
    assert rel_err(final, g["meta_theta_final"]) < 5e-3   # chained Adam steps, sign flips at g~0 allowed
    np.testing.assert_allclose(np.stack(es._archive), g["archive_final"], rtol=1e-3, atol=1e-4)
    assert abs(es.best_reward - float(max(g["episode_reward"]))) < 1e-4


# ------------------------------------------------------------------ fused mode for every combination
class _Spy(OracleBackend):
    def __init__(self, **kw):
        super().__init__(**kw)
        self.acts = set()

    def eval_mlp(self, *a, **kw):
        self.acts.add(kw.get("act", 0))
        return super().eval_mlp(*a, **kw)

    def eval_mlp_center(self, *a, **kw):
        self.acts.add(kw.get("act", 0))
        return super().eval_mlp_center(*a, **kw)


@pytest.mark.parametrize("hidden,output", [("relu", "identity"), ("tanh", "identity"), ("relu", "tanh"),
                                           ("tanh", "tanh")])
@pytest.mark.parametrize("tensor_core", [False, True])
def test_fused_for_every_combination_and_the_code_reaches_the_kernels(hidden, output, tensor_core):
    dims, B = ([64, 64, 32], 256) if tensor_core else ([4, 16, 2], 8)
    rng = np.random.RandomState(3)
    obs = torch.from_numpy(rng.standard_normal((B, dims[0])).astype(np.float32))
    tgt = torch.from_numpy(rng.uniform(-0.9, 0.9, (B, dims[-1])).astype(np.float32))
    be = _Spy(tensor_core=tensor_core)
    es = E.ES(ActMLP, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
              policy_kwargs={"dims": dims, "hidden": hidden, "output": output},
              agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 16,
              _backend=be)
    es.log = lambda: None
    assert es._fused and es._spec.act == mlp.code(hidden, output)
    assert es._precision == ("f16" if tensor_core else "fp32")       # "auto" picks f16 where the shape allows
    es.train(n_steps=3)
    assert be.acts == {mlp.code(hidden, output)}
    # the trained policy's own forward agrees with the fused episode reward
    with torch.no_grad():
        want = float(-((es.policy(obs) - tgt) ** 2).mean())
    fwd = mlp.FORWARD[es._precision]
    emu = float(orc.synthetic_return(fwd(es._slots[0].theta.numpy(), dims, obs.numpy(), hidden, output), tgt.numpy()))
    assert abs(es.episode_reward - emu) < 1e-6 * abs(emu) + 1e-7
    assert abs(es.episode_reward - want) < (1e-5 if not tensor_core else 1e-4) * abs(want)


def test_gelu_policy_stays_in_hooks_mode():
    es = E.ES(ActMLP, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
              policy_kwargs={"dims": [4, 16, 2], "hidden": "gelu"},
              agent_kwargs=dict(obs=torch.randn(8, 4), target=torch.randn(8, 2)), noise_table_size=1 << 12,
              _backend=OracleBackend())
    assert es._spec is None and not es._fused
