"""Population mode of a generic convolutional policy (a PopulationAgent that declares ``obs_shape``) without a GPU:
recognition, the global RNG stream, mode selection, one act launch per step and the member order of ``act``, the
reference goldens through ES / NSR-ES on the oracle stand-in (tests/_pop_cnn_oracle.py), population mode against
hooks mode, checkpoint / resume, and estk_act_cnn's header, binding and refusals."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import estorch_b200.estorch as E
from estorch_b200 import SequenceAgent, _capi
from estorch_b200.policy_spec import CNNSpec, cnn_spec_from_module
from conftest import ROOT, load_golden, rel_err
from oracle import es_oracle as orc
from _cnn_oracle import forward, pack, policy_class
from _pop_cnn_oracle import (DIMS, ES_POLICY, NSR_POLICY, OBS_SHAPE, PixelPoint, PopCnnOracleBackend,
                             cnn_policy)

CODE = 0 | (1 << 8) | (2 << 24)        # ReLU hidden, Tanh output, two convs (ES_POLICY)


def _es(cls=E.ES, optimizer=torch.optim.Adam, P=8, bc_dim=0, agent=PixelPoint, policy=ES_POLICY, horizon=3,
        backend=None, **kw):
    es = cls(cnn_policy(**policy), agent, optimizer, population_size=P, sigma=0.05, policy_kwargs={"dims": DIMS},
             agent_kwargs={"horizon": horizon, "bc_dim": bc_dim}, optimizer_kwargs={"lr": 0.01},
             noise_table_size=1 << 14, _backend=backend or PopCnnOracleBackend(), **kw)
    es.log = lambda: None
    return es


class _NoShape(PixelPoint):
    obs_shape = None


class _WrongShape(PixelPoint):
    obs_shape = (3, 8, 8)          # the first conv takes 2 channels


# ------------------------------------------------------------------ recognition
def test_obs_shape_makes_the_policy_recognised():
    es = _es()
    assert es._is_cnn and es._population and es._fused
    assert es._spec == CNNSpec(OBS_SHAPE, ((4, 3, 1, 1), (8, 3, 2, 0)), (16, 2), "relu", "tanh")
    assert es._spec.act == CODE
    es = _es(agent=_NoShape)
    assert es._spec is None and not es._fused and not es._population


def test_the_global_rng_is_untouched_and_existing_specs_unchanged():
    torch.manual_seed(3)
    pol = cnn_policy(**NSR_POLICY)(DIMS)
    after_init = torch.get_rng_state()
    assert cnn_spec_from_module(pol, OBS_SHAPE) is not None
    assert torch.equal(torch.get_rng_state(), after_init)
    # ES draws the same global stream with and without obs_shape: the recogniser draws from its own generator
    states = []
    for agent in (PixelPoint, _NoShape):
        torch.manual_seed(3)
        _es(agent=agent)
        states.append(torch.rand(5))
    assert torch.equal(states[0], states[1])
    # the population agents of the MLP, conv + VBN and recurrent policies keep their specs with obs_shape set
    from _pop_oracle import LinearWalker
    from test_api_cpu import MLP

    class ShapedWalker(LinearWalker):
        obs_shape = (1, 4, 6)
    es = E.ES(MLP, ShapedWalker, torch.optim.Adam, population_size=8, sigma=0.05, policy_kwargs={"dims": [24, 8, 4]},
              agent_kwargs={"horizon": 2}, noise_table_size=1 << 13, _backend=PopCnnOracleBackend())
    assert type(es._spec).__name__ == "MLPSpec" and not es._is_cnn


# ------------------------------------------------------------------ mode selection and launch counts
@pytest.mark.parametrize("cls,bc_dim", [(E.ES, 0), (E.NS_ES, 4), (E.NSR_ES, 4), (E.NSRA_ES, 4)])
def test_population_mode_is_selected_and_counts_its_launches(cls, bc_dim):
    es = _es(cls=cls, bc_dim=bc_dim)
    assert es._fused and es._population and es._is_cnn and es._precision == "fp32"
    assert es.agent.device == es._dev
    be = es._be
    meta = len(es._slots) if bc_dim else 0
    a0 = be.cnn_act_calls
    assert a0 == 3 * meta                         # NS family: the archive's initial centre rollouts
    es.train(n_steps=2)
    # per generation: 3 steps of the population and 3 of theta's rollout; the NS family with a meta-population
    # also rolls out each member when it picks one (estorch.py:444-456)
    per_gen = 2 + (meta if cls in (E.NSR_ES, E.NSRA_ES, E.NS_ES) else 0)
    assert be.cnn_act_calls - a0 == 2 * 3 * per_gen
    assert be.act_calls == 0


class _OwnReturns(E.ES):
    def _calculate_returns(self, parameters):
        return super()._calculate_returns(parameters)


@pytest.mark.parametrize("case", ["sgd", "overridden_hook", "two_workers", "sequence_agent", "wrong_shape"])
def test_hooks_mode_serves_everything_else(case, monkeypatch):
    kw = {}
    if case == "sgd":
        kw["optimizer"] = torch.optim.SGD
    elif case == "overridden_hook":
        kw["cls"] = _OwnReturns
    elif case == "two_workers":
        monkeypatch.setenv("WORLD_SIZE", "2")
        monkeypatch.setenv("RANK", "0")
    elif case == "wrong_shape":
        kw["agent"] = _WrongShape
    if case == "sequence_agent":
        # a SequenceAgent holds [B, T, in] sequences, no images: the CNN is not recognised for it, and a CNN spec
        # would still be refused
        g = torch.Generator().manual_seed(4)
        es = E.ES(cnn_policy(**ES_POLICY), SequenceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
                  policy_kwargs={"dims": DIMS}, noise_table_size=1 << 14, _backend=PopCnnOracleBackend(),
                  agent_kwargs=dict(obs=torch.randn(3, 2, 128, generator=g), target=torch.randn(3, 2, 2, generator=g)))
        assert not es._fused and not es._is_cnn
        es._spec = CNNSpec(OBS_SHAPE, ((4, 3, 1, 1), (8, 3, 2, 0)), (16, 2), "relu", "tanh")
        es._is_cnn = True
        assert not es._decide_fused(torch.optim.Adam)
        return
    es = _es(**kw)
    assert not es._fused and not es._population
    assert es.agent.device == es.device
    if case != "two_workers":
        es.train(n_steps=1)
        assert es._be.cnn_act_calls == 0


@pytest.mark.parametrize("bad", [(2, 8), (2, 8, 0), (2, 8.0, 8), (2, True, 8), "2x8x8", (2, 8, 8, 1), (-2, 8, 8)])
def test_a_malformed_obs_shape_is_refused(bad):
    class Bad(PixelPoint):
        obs_shape = bad
    with pytest.raises(ValueError, match="obs_shape"):
        _es(agent=Bad)
    class Listed(PixelPoint):
        obs_shape = [2, 8, 8]
    assert _es(agent=Listed)._population


@pytest.mark.parametrize("precision", ["f16", "bf16"])
def test_population_mode_refuses_a_tensor_core_precision(precision):
    with pytest.raises(ValueError, match="fp32 only"):
        _es(eval_precision=precision)
    assert _es(eval_precision="fp32")._population


# ------------------------------------------------------------------ act
def _rows(es, slot):
    rows, _ = orc.sample_population(slot.theta_prev.numpy(), es._table.numpy(), es._offsets.numpy(), es.sigma)
    return rows


def test_act_member_order_shapes_and_one_launch_per_call():
    es = _es(P=6)
    slot = es._slots[0]
    slot.theta_prev.copy_(slot.theta)
    es._draw_offsets()
    act = es._population_act(slot)
    pts = torch.from_numpy(np.random.RandomState(0).uniform(-0.8, 0.8, (12, 2)).astype(np.float32))
    obs = PixelPoint().frames(pts).numpy().reshape(6, 2, *OBS_SHAPE)
    n0 = es._be.cnn_act_calls
    out = act(torch.from_numpy(obs)).numpy()
    assert es._be.cnn_act_calls == n0 + 1
    assert out.shape == (6, 2, 2)
    rows = _rows(es, slot)
    # row i < P/2 is theta + sigma*T[off_i], row P/2 + i its mirror, each on its own images
    for m in range(6):
        np.testing.assert_array_equal(out[m], forward(rows[m], DIMS, CODE, obs[m]))
        pol = cnn_policy(**ES_POLICY)(DIMS)
        torch.nn.utils.vector_to_parameters(torch.from_numpy(rows[m]), pol.parameters())
        with torch.no_grad():
            want = pol(torch.from_numpy(obs[m])).numpy()
        assert np.abs(out[m] - want).max() <= 1e-5 * np.abs(want).max()
    single = act(torch.from_numpy(obs[:, 0])).numpy()
    assert single.shape == (6, 2) and es._be.cnn_act_calls == n0 + 2
    for m in range(6):
        np.testing.assert_array_equal(single[m], forward(rows[m], DIMS, CODE, obs[m, :1])[0])
    centre = es._population_act(slot, centre=True)
    th = slot.theta.numpy()
    np.testing.assert_array_equal(centre(torch.from_numpy(obs[:1, 0])).numpy()[0],
                                  forward(th, DIMS, CODE, obs[0, :1])[0])
    np.testing.assert_array_equal(centre(torch.from_numpy(obs[:1])).numpy()[0], forward(th, DIMS, CODE, obs[0]))
    for bad in (torch.zeros(5, *OBS_SHAPE), torch.zeros(6, 3, 8, 8), torch.zeros(6, 8, 8), torch.zeros(6, 2, 2, 8, 7)):
        with pytest.raises(ValueError, match=r"expected \[6, 2, 8, 8\] or \[6, B, 2, 8, 8\]"):
            act(bad)


def test_rollout_is_the_reference_protocol():
    ag = PixelPoint(horizon=3)
    pol = cnn_policy(**ES_POLICY)(DIMS)
    r = ag.rollout(pol)
    with torch.no_grad():
        ret = ag.rollout_population(lambda o: pol(o), 1)
    assert isinstance(r, float) and r == float(ret[0])
    r2, bc = PixelPoint(horizon=4, bc_dim=4).rollout(pol)
    assert isinstance(r2, float) and bc.shape == (4,)


# ------------------------------------------------------------------ the reference goldens
class _Rec:
    def log(self):
        self.rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                             best=self.best_reward, idx=getattr(self, "idx", None),
                             archive=len(getattr(self, "_archive", []))))


def _load_theta(module, flat):
    torch.nn.utils.vector_to_parameters(torch.from_numpy(np.asarray(flat, np.float32).copy()), module.parameters())


def _golden_es(cls, g, backend, policy, **kw):
    class R(_Rec, cls):
        pass
    es = R(cnn_policy(**policy), PixelPoint, torch.optim.Adam, population_size=int(g["P"]), sigma=float(g["sigma"]),
           policy_kwargs={"dims": DIMS}, optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]),
           noise_seed=int(g["noise_seed"]), _backend=backend, **kw)
    es.rec = []
    assert es._population and es._is_cnn
    assert tuple(int(d) for d in g["dims"]) == tuple(DIMS)
    es._table.copy_(torch.from_numpy(g["table"]).to(es._dev))
    return es


def run_es_golden(backend):
    """ES in population mode from es_pop_cnn_p16.npz's start; returns (instance, fixture)."""
    g = load_golden("es_pop_cnn_p16.npz")
    es = _golden_es(E.ES, g, backend, ES_POLICY)
    _load_theta(es.policy, g["theta0"])
    es._slots[0].ensure_flat()
    es.train(n_steps=len(g["returns"]))
    return es, g


def check_es_golden(es, g):
    for gen in range(len(g["returns"])):
        assert rel_err(es.rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-5
        assert abs(es.rec[gen]["episode"] - float(g["episode_reward"][gen])) < 1e-5 * abs(float(g["episode_reward"][gen]))
        assert abs(es.rec[gen]["best"] - float(g["best_reward"][gen])) < 1e-5 * abs(float(g["best_reward"][gen]))
    theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().cpu().numpy()
    assert rel_err(theta, g["theta_after"][-1]) < 2e-4
    bp = es.best_policy_dict
    best = np.concatenate([v.reshape(-1).cpu().numpy() for v in bp.values()])
    assert rel_err(best, g["best_theta"]) < 2e-4


def run_nsr_golden(backend):
    g = load_golden("nsr_pop_cnn_p8.npz")
    np.random.seed(123)
    es = _golden_es(E.NSR_ES, g, backend, NSR_POLICY, agent_kwargs={"bc_dim": 4}, k=int(g["k"]))
    for i, (p, _) in enumerate(es.meta_population):
        _load_theta(p, g["meta_theta0"][i])
        es._slots[i].ensure_flat()
        es._slots[i].push_theta()
    es._archive = [a.copy() for a in g["archive0"]]
    np.random.seed(123)
    es.train(n_steps=len(g["returns"]))
    return es, g


def check_nsr_golden(es, g):
    for gen in range(len(g["returns"])):
        r = es.rec[gen]
        assert r["idx"] == int(g["idx"][gen])
        assert rel_err(r["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-5
        assert rel_err(r["returns"][:, 1], g["returns"][gen][:, 1]) < 1e-3
        assert abs(r["episode"] - float(g["episode_reward"][gen])) < 1e-5 * abs(float(g["episode_reward"][gen]))
        assert r["archive"] == int(g["archive_len"][gen])
    np.testing.assert_allclose(np.stack(es._archive), g["archive_final"], rtol=1e-4, atol=1e-6)


def test_es_population_mode_matches_reference_golden():
    check_es_golden(*run_es_golden(PopCnnOracleBackend()))


def test_nsr_population_mode_matches_reference_golden():
    check_nsr_golden(*run_nsr_golden(PopCnnOracleBackend()))


# ------------------------------------------------------------------ population mode against hooks mode
class _Hooks(E.ES):
    def _after_optimize(self, policy):          # any overridden hook selects hooks mode
        super()._after_optimize(policy)


def test_population_mode_matches_hooks_mode_on_the_same_agent():
    runs = []
    for cls in (E.ES, _Hooks):
        torch.manual_seed(5)
        es = _es(cls=cls, P=6)
        rec = []
        es.log = lambda es=es, rec=rec: rec.append((es.population_returns.copy(), es.episode_reward))
        es.train(n_steps=2)
        theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().numpy()
        runs.append((es._population, rec, theta))
    (pop_mode, pop_rec, pop_theta), (hooks_mode, hooks_rec, hooks_theta) = runs
    assert pop_mode and not hooks_mode
    for (rp, ep), (rh, eh) in zip(pop_rec, hooks_rec):
        assert rel_err(rp[:, 0], rh[:, 0]) < 1e-5
        assert abs(ep - eh) < 1e-5 * abs(eh)
    assert rel_err(pop_theta, hooks_theta) < 2e-4


# ------------------------------------------------------------------ checkpoint / resume
@pytest.mark.parametrize("cls,bc_dim", [(E.ES, 0), (E.NSR_ES, 4)])
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


# ------------------------------------------------------------------ ABI: header, binding, refusals
def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


def test_act_cnn_is_declared_apart_from_the_core_header_and_bound_to_it():
    header = open(os.path.join(ROOT, "include", "estk_act_cnn.h")).read()
    assert '#include "estk.h"' in header
    declared = sorted(set(re.findall(r"ESTK_API\s+[\w\s\*]+?\b(estk_\w+)\s*\(", header)))
    assert declared == sorted(_capi.ACT_CNN_SIGNATURES) == ["estk_act_cnn"]
    m = re.search(r"\bestk_act_cnn\s*\(([^)]*)\)", header)
    assert len(m.group(1).split(",")) == len(_capi.ACT_CNN_SIGNATURES["estk_act_cnn"]) == 13
    for text in ("ESTK_ACTIONS", "ESTK_ERR_INVALID", "bit for bit", "64-bit", "ESTK_MAX_POPULATION/2"):
        assert text in header, text
    core = open(os.path.join(ROOT, "include", "estk.h")).read()
    assert "estk_act_cnn" not in core and re.search(r"#define\s+ESTK_VERSION\s+200\b", core)
    assert "estk_act_cnn" not in _capi.SIGNATURES and "estk_act_cnn" not in _capi.BATCH_SIGNATURES
    lib = _lib()
    assert lib.estk_act_cnn.argtypes is not None


FAKE = C.c_void_p(256)          # never dereferenced: every call below is refused before the context is read
SMALL = pack((1, 6, 6), [(2, 3, 1, 0)], [3])          # conv 1->2 k3 -> 2x4x4 -> Linear 3
SMALL_CODE = 3 << 16 | 1 << 24


def _act_cnn(centre=False, **over):
    """estk_act_cnn on a well-formed call (pairs = 2, B = 1) with the arguments in ``over`` replaced; the outputs
    are host arrays that a refused call must leave untouched.  Returns (status, outputs unchanged)."""
    dims = over.pop("dims", SMALL)
    d = _capi.EstkMlpDesc()
    d.n_layers = over.pop("n_layers", len(dims) - 1)
    for i, w in enumerate(dims):
        d.dims[i] = C.c_int32(int(w)).value
    d.activation = C.c_int32(int(over.pop("code", SMALL_CODE))).value
    buf = np.full(64, 7.0, np.float32)
    ptr = lambda a: C.c_void_p(a.ctypes.data)       # noqa: E731
    th, tab, obs = np.zeros(64, np.float32), np.zeros(4096, np.float32), np.zeros(4 * 36, np.float32)
    off, order = np.zeros(2, np.int64), np.zeros(2, np.int32)
    args = dict(ctx=FAKE, desc=C.byref(d), theta=ptr(th), table=ptr(tab), offsets=None if centre else ptr(off),
                order=ptr(order), pairs=2, sigma=0.1, obs=ptr(obs), B=1, out_plus=ptr(buf[:32]),
                out_minus=ptr(buf[32:]), stream=None)
    args.update(over)
    rc = _lib().estk_act_cnn(*args.values())
    return rc, bool((buf == 7.0).all())


@pytest.mark.parametrize("centre", [False, True])
@pytest.mark.parametrize("over", [
    dict(ctx=None), dict(desc=None), dict(theta=None), dict(obs=None), dict(out_plus=None), dict(B=0), dict(B=-3),
    dict(code=SMALL_CODE & ~(0xff << 24)), dict(code=SMALL_CODE | 8 << 24), dict(code=(SMALL_CODE & ~(3 << 16))),
    dict(code=(SMALL_CODE & ~(3 << 16)) | 1 << 16), dict(code=(SMALL_CODE & ~(3 << 16)) | 2 << 16),
    dict(code=SMALL_CODE | 8), dict(code=SMALL_CODE | 9), dict(code=SMALL_CODE | 2), dict(code=SMALL_CODE | 6),
    dict(code=SMALL_CODE | 2 << 8), dict(code=SMALL_CODE | 0x1000),
    dict(n_layers=1), dict(n_layers=9), dict(dims=pack((0, 6, 6), [(2, 3, 1, 0)], [3])),
    dict(dims=(SMALL[0] | 1 << 30,) + SMALL[1:]), dict(dims=pack((1, 6, 6), [(0, 3, 1, 0)], [3])),
    dict(dims=pack((1, 6, 6), [(2, 3, 1, 3)], [3])), dict(dims=pack((1, 6, 6), [(2, 0, 1, 0)], [3])),
    dict(dims=pack((1, 6, 6), [(2, 3, 0, 0)], [3])), dict(dims=pack((1, 2, 2), [(2, 5, 1, 1)], [3])),
    dict(dims=pack((1, 6, 6), [(2, 3, 1, 0)], [0])),
    dict(dims=pack((1, 1023, 1023), [(4095, 1, 1, 0)], [3])),     # more than 2^30 outputs per image
])
def test_refusals_are_invalid_before_any_launch(centre, over):
    rc, untouched = _act_cnn(centre=centre, **over)
    assert rc == -1 and untouched, _lib().estk_last_error().decode()


@pytest.mark.parametrize("over", [dict(table=None), dict(out_minus=None), dict(pairs=0),
                                  dict(pairs=(1 << 21) + 1), dict(pairs=-1)])
def test_population_refusals_are_invalid(over):
    rc, untouched = _act_cnn(**over)
    assert rc == -1 and untouched, _lib().estk_last_error().decode()
