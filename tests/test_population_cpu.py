"""Population mode (estorch_b200.PopulationAgent) without a GPU: mode selection, the member order of
``act``, the reference goldens reproduced through ES / NSR-ES on the oracle stand-in
(tests/_oracle_backend.py), population mode against hooks mode, checkpoint / resume, the multi-GPU fallback,
and the ESTK_ACTIONS code in the header, the binding and the library's support probe."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import estorch_b200.estorch as E
from estorch_b200 import PopulationAgent, _capi
from conftest import ROOT, load_golden, rel_err
from oracle import es_oracle as orc
from _mlp_oracle import ACTIONS, MLP, act_forward
from _oracle_backend import OracleBackend
from _pop_oracle import LinearWalker

DIMS = [24, 64, 64, 4]


def _es(cls=E.ES, optimizer=torch.optim.Adam, policy=MLP, P=16, bc_dim=0, backend=None, **kw):
    es = cls(policy, LinearWalker, optimizer, population_size=P, sigma=0.05,
             policy_kwargs={"dims": DIMS, "hidden": "relu", "output": "tanh"} if policy is MLP else {},
             agent_kwargs={"horizon": 6, "bc_dim": bc_dim}, optimizer_kwargs={"lr": 0.01},
             noise_table_size=1 << 16, _backend=backend or OracleBackend(), **kw)
    es.log = lambda: None
    return es


# ------------------------------------------------------------------ mode selection
def test_population_mode_is_selected_for_a_population_agent():
    es = _es()
    assert es._fused and es._population and es._precision == "fp32"
    assert es.agent.device == es._dev
    es.train(n_steps=2)
    assert es._be.act_calls == 2 * (6 + 6)        # population and centre episodes, 6 steps each


class _Unrecognised(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(24, 4)

    def forward(self, x):
        return torch.sigmoid(self.lin(x))


class _OwnReturns(E.ES):
    def _calculate_returns(self, parameters):
        return super()._calculate_returns(parameters)


@pytest.mark.parametrize("case", ["sgd", "unrecognised_policy", "overridden_hook", "two_workers"])
def test_hooks_mode_serves_everything_else(case, monkeypatch):
    kw = {}
    if case == "sgd":
        kw["optimizer"] = torch.optim.SGD
    elif case == "unrecognised_policy":
        kw["policy"] = _Unrecognised
    elif case == "overridden_hook":
        kw["cls"] = _OwnReturns
    else:                  # multi-GPU population generations are not implemented: hooks mode serves them
        monkeypatch.setenv("WORLD_SIZE", "2")
        monkeypatch.setenv("RANK", "0")
    es = _es(**kw)
    assert not es._fused and not es._population
    assert es.agent.device == es.device
    if case != "two_workers":
        es.train(n_steps=1)
        assert es._be.act_calls == 0


@pytest.mark.parametrize("precision", ["f16", "bf16", "bf16s"])
def test_population_mode_refuses_a_tensor_core_precision(precision):
    with pytest.raises(ValueError, match="fp32 only"):
        _es(eval_precision=precision)
    assert _es(eval_precision="fp32")._population


# ------------------------------------------------------------------ act
def test_act_member_order_and_shapes():
    es = _es(P=8)
    slot = es._slots[0]
    slot.theta_prev.copy_(slot.theta)
    es._draw_offsets()
    act = es._population_act(slot)
    rng = np.random.RandomState(0)
    obs = rng.standard_normal((8, 3, 24)).astype(np.float32)
    out = act(torch.from_numpy(obs)).numpy()
    rows, _ = orc.sample_population(slot.theta.numpy(), es._table.numpy(), es._offsets.numpy(), es.sigma)
    np.testing.assert_array_equal(out, act_forward(rows, DIMS, obs, slot_code(es)))
    # row i < P/2 is theta + sigma*T[off_i], row P/2 + i its mirror, each on its own observations
    for m in (0, 3, 4, 7):
        policy = MLP(DIMS, "relu", "tanh")
        torch.nn.utils.vector_to_parameters(torch.from_numpy(rows[m]), policy.parameters())
        np.testing.assert_allclose(out[m], policy(torch.from_numpy(obs[m])).detach().numpy(), rtol=0, atol=2e-6)
    single = act(torch.from_numpy(obs[:, 0])).numpy()
    np.testing.assert_array_equal(single, out[:, 0])
    centre = es._population_act(slot, centre=True)(torch.from_numpy(obs[:1, 0])).numpy()
    np.testing.assert_array_equal(centre, act_forward(slot.theta.numpy()[None], DIMS, obs[:1, :1], slot_code(es))[:, 0])
    with pytest.raises(ValueError, match="expected"):
        act(torch.zeros(7, 24))


def slot_code(es):
    return es._spec.act | ACTIONS


def test_rollout_is_the_reference_protocol():
    ag = LinearWalker(horizon=5)
    pol = MLP(DIMS, "relu", "tanh")
    r = ag.rollout(pol)
    assert isinstance(r, float)
    with torch.no_grad():
        ret = ag.rollout_population(lambda o: pol(o), 1)
    assert r == float(ret[0])
    r2, bc = LinearWalker(horizon=6, bc_dim=48).rollout(pol)
    assert isinstance(r2, float) and bc.shape == (48,)
    with pytest.raises(NotImplementedError):
        PopulationAgent().rollout(pol)


# ------------------------------------------------------------------ the reference goldens
class _Rec:
    def log(self):
        self.rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                             best=self.best_reward, idx=getattr(self, "idx", None),
                             archive=len(getattr(self, "_archive", []))))


def _load_theta(module, flat):
    torch.nn.utils.vector_to_parameters(torch.from_numpy(flat.copy()), module.parameters())


def run_es_golden(backend):
    """ES in population mode from es_pop_walker_p64.npz's start; returns (instance, fixture)."""
    g = load_golden("es_pop_walker_p64.npz")

    class R(_Rec, E.ES):
        pass
    es = R(MLP, LinearWalker, torch.optim.Adam, population_size=64, sigma=float(g["sigma"]),
           policy_kwargs={"dims": DIMS, "hidden": "relu", "output": "tanh"}, optimizer_kwargs={"lr": 0.01},
           noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]), _backend=backend)
    es.rec = []
    assert es._population
    es._table.copy_(torch.from_numpy(g["table"]).to(es._dev))
    _load_theta(es.policy, g["theta0"])
    es._slots[0].ensure_flat()
    es.train(n_steps=3)
    return es, g


def check_es_golden(es, g):
    for gen in range(3):
        assert rel_err(es.rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-5
        assert abs(es.rec[gen]["episode"] - float(g["episode_reward"][gen])) < 1e-5 * abs(float(g["episode_reward"][gen]))
        assert abs(es.rec[gen]["best"] - float(g["best_reward"][gen])) < 1e-5 * abs(float(g["best_reward"][gen]))
    theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().cpu().numpy()
    assert rel_err(theta, g["theta_after"][2]) < 2e-4
    bp = es.best_policy_dict
    assert rel_err(np.concatenate([v.reshape(-1).cpu().numpy() for v in bp.values()]), g["best_theta"]) < 2e-4


def run_nsr_golden(backend):
    g = load_golden("nsr_pop_walker_p32.npz")

    class R(_Rec, E.NSR_ES):
        pass
    np.random.seed(123)
    es = R(MLP, LinearWalker, torch.optim.Adam, population_size=32, sigma=float(g["sigma"]),
           policy_kwargs={"dims": DIMS, "hidden": "relu", "output": "tanh"}, agent_kwargs={"bc_dim": 48},
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]),
           _backend=backend)
    es.rec = []
    assert es._population
    es._table.copy_(torch.from_numpy(g["table"]).to(es._dev))
    for i, (p, _) in enumerate(es.meta_population):
        _load_theta(p, g["meta_theta0"][i])
        es._slots[i].ensure_flat()
        es._slots[i].push_theta()
    es._archive = [a.copy() for a in g["archive0"]]
    np.random.seed(123)
    es.train(n_steps=len(g["grad"]))
    return es, g


def check_nsr_golden(es, g):
    for gen in range(len(g["grad"])):
        r = es.rec[gen]
        assert r["idx"] == int(g["idx"][gen])
        assert rel_err(r["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-5
        assert rel_err(r["returns"][:, 1], g["returns"][gen][:, 1]) < 1e-4
        assert abs(r["episode"] - float(g["episode_reward"][gen])) < 1e-5 * abs(float(g["episode_reward"][gen]))
        assert r["archive"] == int(g["archive_len"][gen])
    np.testing.assert_allclose(np.stack(es._archive), g["archive_final"], rtol=1e-3, atol=1e-5)


def test_es_population_mode_matches_reference_golden():
    check_es_golden(*run_es_golden(OracleBackend()))


def test_nsr_population_mode_matches_reference_golden():
    check_nsr_golden(*run_nsr_golden(OracleBackend()))


# ------------------------------------------------------------------ population mode against hooks mode
class _Hooks(E.ES):
    def _after_optimize(self, policy):          # any overridden hook selects hooks mode
        super()._after_optimize(policy)


def test_population_mode_matches_hooks_mode_on_the_same_agent():
    runs = []
    for cls in (E.ES, _Hooks):
        torch.manual_seed(5)
        es = _es(cls=cls, P=8)
        rec = []
        es.log = lambda es=es, rec=rec: rec.append((es.population_returns.copy(), es.episode_reward))
        es.train(n_steps=3)
        theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().numpy()
        runs.append((es._population, rec, theta))
    (pop_mode, pop_rec, pop_theta), (hooks_mode, hooks_rec, hooks_theta) = runs
    assert pop_mode and not hooks_mode
    for (rp, ep), (rh, eh) in zip(pop_rec, hooks_rec):
        assert rel_err(rp[:, 0], rh[:, 0]) < 1e-5
        assert abs(ep - eh) < 1e-5 * abs(eh)
    assert rel_err(pop_theta, hooks_theta) < 2e-4


# ------------------------------------------------------------------ checkpoint / resume
@pytest.mark.parametrize("cls,bc_dim", [(E.ES, 0), (E.NSR_ES, 48)])
def test_checkpoint_resume_is_bit_identical(cls, bc_dim):
    torch.manual_seed(1)
    np.random.seed(1)
    a = _es(cls=cls, bc_dim=bc_dim)
    a.train(n_steps=3)
    torch.manual_seed(1)
    np.random.seed(1)
    b = _es(cls=cls, bc_dim=bc_dim)
    b.train(n_steps=2)
    sd = b.state_dict()
    torch.manual_seed(99)
    c = _es(cls=cls, bc_dim=bc_dim)
    c.load_state_dict(sd)
    c.train(n_steps=1)
    for sa, sc in zip(a._slots, c._slots):
        assert torch.equal(sa.theta, sc.theta) and torch.equal(sa.m, sc.m) and torch.equal(sa.v, sc.v)
    assert a.best_reward == c.best_reward
    np.testing.assert_array_equal(a.population_returns, c.population_returns)


# ------------------------------------------------------------------ ABI
def test_header_and_binding_agree_on_actions():
    header = open(os.path.join(ROOT, "include", "estk.h")).read()
    m = re.search(r"#define\s+ESTK_ACTIONS\s+\((\d+)\s*<<\s*16\)", header)
    assert m and int(m.group(1)) << 16 == _capi.ESTK_ACTIONS == ACTIONS == 0x30000
    assert re.search(r"#define\s+ESTK_VERSION\s+200\b", header)
    assert not re.search(r"#define\s+ESTK_\w+\s+\(2\s*<<\s*16\)", header)       # loss value 2 stays undefined


def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


ACTION_CODES = [h | o | ACTIONS for h in (0, 1, 3, 4, 5) for o in (0, 1 << 8)]
REFUSED = [2, 0xff, 0x200, -1, 1 << 24, 0x20000, 0x10200, 6, 0x0102, 0x10002, 0x30002, 0x30006, 0x40000,
           0x30200, 0x70000] + [0x10100 | h for h in (0, 1, 3, 4, 5)]


def test_support_probe_refuses_the_action_codes_under_every_precision():
    from estorch_b200.backend import mlp_desc
    lib = _lib()
    sup = lambda dims, code, prec, B: lib.estk_eval_mlp_supported(C.byref(mlp_desc(dims, code)), prec, B)  # noqa
    precs = (_capi.ESTK_PREC_FP32, _capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S,
             _capi.ESTK_PREC_F16_ANY)
    for code in ACTION_CODES + REFUSED:
        for prec in precs:
            assert sup([64, 64, 32], code, prec, 256) == 0, (hex(code), prec)
        assert sup([784, 100, 10], code, _capi.ESTK_PREC_F16_ANY, 100) == 0, hex(code)
    for code in (0, 0x100, 0x10000, 5 | 0x100):          # the codes that compute a return are served as before
        assert sup([64, 64, 32], code, _capi.ESTK_PREC_F16, 256) == 1
        assert sup([784, 100, 10], code, _capi.ESTK_PREC_F16_ANY, 100) == 1
