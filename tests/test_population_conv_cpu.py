"""Population mode of the conv + VirtualBatchNorm policy without a GPU: mode selection, one stats launch per
generation and per centre rollout and one act launch per step, the member order of ``act``, the reference
goldens reproduced through ES / NSR-ES on the oracle stand-in (tests/_pop_conv_oracle.py), population mode
against hooks mode, checkpoint / resume, and the action mode in the header."""
import os
import re

import numpy as np
import pytest
import torch

import estorch_b200.estorch as E
from estorch_b200 import _capi
from conftest import ROOT, load_golden, rel_err
from oracle import es_oracle as orc
from _oracle_backend import OracleBackend
from _pop_conv_oracle import (STATS_FLOATS, AtariPolicy, PixelWalker, conv_act, conv_stats,
                              golden_table, golden_theta0, theta_subset, walker_xref)

A = 4


def _es(cls=E.ES, optimizer=torch.optim.Adam, P=8, bc_dim=0, backend=None, horizon=3, **kw):
    es = cls(AtariPolicy, PixelWalker, optimizer, population_size=P, sigma=0.05,
             policy_kwargs={"n_actions": A, "xref": walker_xref(4)}, agent_kwargs={"horizon": horizon, "bc_dim": bc_dim},
             optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 20, _backend=backend or OracleBackend(),
             **kw)
    es.log = lambda: None
    return es


# ------------------------------------------------------------------ mode selection and launch counts
@pytest.mark.parametrize("cls,bc_dim", [(E.ES, 0), (E.NSR_ES, 4)])
def test_population_mode_is_selected_and_counts_its_launches(cls, bc_dim):
    es = _es(cls=cls, bc_dim=bc_dim)
    assert es._fused and es._population and es._is_conv and es._precision == "fp32"
    assert es.agent.device == es._dev
    assert tuple(es._conv_stats.shape) == (8, STATS_FLOATS)
    be = es._be
    s0, a0 = be.stats_calls, be.conv_act_calls
    meta = len(es._slots) if bc_dim else 0
    assert (s0, a0) == (meta, 3 * meta)                     # NS family: the archive's initial centre rollouts
    es.train(n_steps=2)
    # per generation: one population stats launch + 3 act launches, and theta's rollout (one stats + 3 acts);
    # NSR-ES also rolls out each meta-population member when it picks one (estorch.py:444-456)
    per_gen = 2 + meta
    assert be.stats_calls - s0 == 2 * per_gen
    assert be.conv_act_calls - a0 == 2 * 3 * per_gen
    assert be.act_calls == 0


class _OwnReturns(E.ES):
    def _calculate_returns(self, parameters):
        return super()._calculate_returns(parameters)


@pytest.mark.parametrize("case", ["sgd", "overridden_hook", "two_workers"])
def test_hooks_mode_serves_everything_else(case, monkeypatch):
    kw = {}
    if case == "sgd":
        kw["optimizer"] = torch.optim.SGD
    elif case == "overridden_hook":
        kw["cls"] = _OwnReturns
    else:
        monkeypatch.setenv("WORLD_SIZE", "2")
        monkeypatch.setenv("RANK", "0")
    es = _es(**kw)
    assert not es._fused and not es._population
    assert es.agent.device == es.device
    if case != "two_workers":
        es.train(n_steps=1)
        assert es._be.stats_calls == es._be.conv_act_calls == 0


@pytest.mark.parametrize("precision", ["f16", "bf16"])
def test_population_mode_refuses_a_tensor_core_precision(precision):
    with pytest.raises(ValueError, match="fp32 only"):
        _es(eval_precision=precision)
    assert _es(eval_precision="fp32")._population


# ------------------------------------------------------------------ act
def _rows_and_stats(es, slot):
    rows, _ = orc.sample_population(slot.theta_prev.numpy(), es._table.numpy(), es._offsets.numpy(), es.sigma)
    return rows, conv_stats(rows, A, es._xref.numpy())


def test_act_member_order_and_shapes():
    es = _es(P=6)
    slot = es._slots[0]
    slot.theta_prev.copy_(slot.theta)
    es._draw_offsets()
    act = es._population_act(slot)
    pts = torch.from_numpy(np.random.RandomState(0).uniform(-0.8, 0.8, (12, 2)).astype(np.float32))
    obs = PixelWalker().frames(pts).numpy().reshape(6, 2, 4, 84, 84)
    out = act(torch.from_numpy(obs)).numpy()
    assert out.shape == (6, 2, A)
    rows, stats = _rows_and_stats(es, slot)
    np.testing.assert_array_equal(out, conv_act(rows, A, stats, obs))
    # row i < P/2 is theta + sigma*T[off_i], row P/2 + i its mirror, each on its own frames
    for m in (0, 2, 3, 5):
        pol = AtariPolicy(A, es._xref)
        torch.nn.utils.vector_to_parameters(torch.from_numpy(rows[m]), pol.parameters())
        with torch.no_grad():
            want = pol(torch.from_numpy(obs[m])).numpy()
        # VBN over 4 reference frames scales near-constant pixels by up to 1/sqrt(1e-5): fp32 order differences
        # between the oracle's products and torch's convolution grow accordingly
        assert np.abs(out[m] - want).max() <= 1e-4 * np.abs(want).max()
    single = act(torch.from_numpy(obs[:, 0])).numpy()
    np.testing.assert_array_equal(single, conv_act(rows, A, stats, obs[:, :1])[:, 0])
    centre = es._population_act(slot, centre=True)(torch.from_numpy(obs[:1, 0])).numpy()
    th = slot.theta.numpy()[None]
    np.testing.assert_array_equal(centre, conv_act(th, A, conv_stats(th, A, es._xref.numpy()), obs[:1, :1])[:, 0])
    for bad in (torch.zeros(5, 4, 84, 84), torch.zeros(6, 3, 84, 84), torch.zeros(6, 84, 84)):
        with pytest.raises(ValueError, match="expected"):
            act(bad)


def test_centre_rollouts_keep_their_own_stats_buffers():
    es = _es(cls=E.NSR_ES, bc_dim=4)
    bufs = [s.conv_stats for s in es._slots]
    assert all(tuple(b.shape) == (1, STATS_FLOATS) for b in bufs)
    assert len({b.data_ptr() for b in bufs} | {es._conv_stats.data_ptr()}) == len(bufs) + 1
    for s, b in zip(es._slots, bufs):
        th = s.theta.numpy()[None]
        np.testing.assert_array_equal(b.numpy(), conv_stats(th, A, es._xref.numpy()))


def test_rollout_is_the_reference_protocol():
    ag = PixelWalker(horizon=3)
    pol = AtariPolicy(A, walker_xref(4))
    r = ag.rollout(pol)
    with torch.no_grad():
        ret = ag.rollout_population(lambda o: pol(o), 1)
    assert isinstance(r, float) and r == float(ret[0])
    r2, bc = PixelWalker(horizon=4, bc_dim=4).rollout(pol)
    assert isinstance(r2, float) and bc.shape == (4,)


# ------------------------------------------------------------------ the reference goldens
class _Rec:
    def log(self):
        self.rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                             best=self.best_reward, idx=getattr(self, "idx", None),
                             archive=len(getattr(self, "_archive", []))))


def _load_theta(module, flat):
    torch.nn.utils.vector_to_parameters(torch.from_numpy(flat.copy()), module.parameters())


def _golden_es(cls, g, backend, **kw):
    class R(_Rec, cls):
        pass
    es = R(AtariPolicy, PixelWalker, torch.optim.Adam, population_size=int(g["P"]), sigma=float(g["sigma"]),
           policy_kwargs={"n_actions": int(g["n_actions"]), "xref": walker_xref(int(g["R"]), int(g["xref_seed"]))},
           optimizer_kwargs={"lr": 0.01}, noise_table_size=int(g["table_len"]), noise_seed=int(g["noise_seed"]),
           _backend=backend, **kw)
    es.rec = []
    assert es._population and es._is_conv
    es._table.copy_(torch.from_numpy(golden_table(int(g["table_len"]), int(g["table_seed"]))).to(es._dev))
    return es


def run_es_golden(backend):
    """ES in population mode from es_pop_conv_p16.npz's start; returns (instance, fixture)."""
    g = load_golden("es_pop_conv_p16.npz")
    es = _golden_es(E.ES, g, backend)
    _load_theta(es.policy, golden_theta0(A, int(g["theta0_seed"])))
    es._slots[0].ensure_flat()
    es.train(n_steps=len(g["returns"]))
    return es, g


def check_es_golden(es, g):
    for gen in range(len(g["returns"])):
        assert rel_err(es.rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-5
        assert abs(es.rec[gen]["episode"] - float(g["episode_reward"][gen])) < 1e-5 * abs(float(g["episode_reward"][gen]))
        assert abs(es.rec[gen]["best"] - float(g["best_reward"][gen])) < 1e-5 * abs(float(g["best_reward"][gen]))
    sub = theta_subset(es.n_parameters)
    theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().cpu().numpy()
    assert rel_err(theta[sub], g["theta_subset_after"]) < 2e-4
    bp = es.best_policy_dict
    best = np.concatenate([v.reshape(-1).cpu().numpy() for v in bp.values()])
    assert rel_err(best[sub], g["best_theta_subset"]) < 2e-4


def run_nsr_golden(backend):
    g = load_golden("nsr_pop_conv_p8.npz")
    np.random.seed(123)
    es = _golden_es(E.NSR_ES, g, backend, agent_kwargs={"bc_dim": 4}, k=int(g["k"]))
    for i, (p, _) in enumerate(es.meta_population):
        _load_theta(p, golden_theta0(A, int(g["meta_seeds"][i])))
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
        # novelty: distances between behaviour characteristics a few hundredths apart, so the BCs' fp32
        # differences (about 1e-6) reach 1e-4 of it
        assert rel_err(r["returns"][:, 1], g["returns"][gen][:, 1]) < 1e-3
        assert abs(r["episode"] - float(g["episode_reward"][gen])) < 1e-5 * abs(float(g["episode_reward"][gen]))
        assert r["archive"] == int(g["archive_len"][gen])
    np.testing.assert_allclose(np.stack(es._archive), g["archive_final"], rtol=1e-4, atol=1e-6)


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


# ------------------------------------------------------------------ ABI
def test_header_documents_the_action_mode():
    header = open(os.path.join(ROOT, "include", "estk.h")).read()
    m = re.search(r"#define\s+ESTK_CONV_VBN_STATS_FLOATS\s+(\d+)", header)
    assert m and int(m.group(1)) == STATS_FLOATS == _capi.ESTK_CONV_VBN_STATS_FLOATS == 2 * 6400 + 2 * 2592
    assert re.search(r"#define\s+ESTK_VERSION\s+200\b", header)
    conv = header[header.index("Action mode (an environment population"):header.index("ESTK_CONV_VBN_STATS_FLOATS 17984")]
    for field in ("bits 0-7", "bits 8-15", "bits 16-23", "ESTK_ACTIONS", "ESTK_ERR_UNSUPPORTED", "table16"):
        assert field in conv, field
