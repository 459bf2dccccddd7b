"""Recurrent policies in population mode without a GPU: recognition of the GRUCell / LSTMCell + Linear head
convention, mode selection, the member order and state of ``act``, the reference goldens reproduced through ES /
NSR-ES on the oracle stand-in (tests/_rnn_oracle.py), population mode against hooks mode, checkpoint / resume,
and the cell codes in the header, the binding and the library's support probe."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import estorch_b200.estorch as E
from estorch_b200 import DeviceAgent, _capi
from estorch_b200.policy_spec import RNNSpec, rnn_spec_from_module
from conftest import ROOT, load_golden, rel_err
from oracle import es_oracle as orc
from _oracle_backend import OracleBackend
from _rnn_oracle import (ACTIONS, CELL_GRU, CELL_LSTM, RecallAgent, param_count, policy_class,
                         state_width, step32)

DIMS = (4, 16, 3)


def _es(cls=E.ES, optimizer=torch.optim.Adam, cell="gru", out_tanh=True, P=16, bc_dim=0, **kw):
    es = cls(policy_class(cell, out_tanh), RecallAgent, optimizer, population_size=P, sigma=0.05,
             policy_kwargs={"dims": DIMS}, agent_kwargs={"bc_dim": bc_dim}, optimizer_kwargs={"lr": 0.01},
             noise_table_size=1 << 14, _backend=OracleBackend(), **kw)
    es.log = lambda: None
    return es


# ------------------------------------------------------------------ recognition
@pytest.mark.parametrize("cell", ["gru", "lstm"])
@pytest.mark.parametrize("out_tanh", [False, True])
def test_recognises_both_cells_with_either_output(cell, out_tanh):
    spec = rnn_spec_from_module(policy_class(cell, out_tanh)(DIMS))
    assert spec == RNNSpec(cell, DIMS, "tanh" if out_tanh else "identity")
    assert spec.n_parameters == param_count(cell, DIMS) == sum(p.numel() for p in policy_class(cell)(DIMS).parameters())
    assert spec.act == (CELL_GRU if cell == "gru" else CELL_LSTM) | (0x100 if out_tanh else 0)
    assert spec.state_width == state_width(cell, DIMS[1])


class _Module(torch.nn.Module):
    """A policy of the given modules whose forward is ``fwd(self, x, state)``."""

    def __init__(self, fwd, **mods):
        super().__init__()
        for k, v in mods.items():
            setattr(self, k, v)
        self._fwd = fwd

    def forward(self, x, state=None):
        return self._fwd(self, x, state)


def _gru_head(m, x, s):
    h = m.cell(x, s)
    return m.head(h), h


def _non_forms():
    G, L, Lin = torch.nn.GRUCell, torch.nn.LSTMCell, torch.nn.Linear
    return {
        "stacked_cells": _Module(lambda m, x, s: (m.head(m.c2(m.cell(x, s))), s), cell=G(4, 16), c2=G(16, 16),
                                 head=Lin(16, 3)),
        "gru_sequence": _Module(lambda m, x, s: (m.head(m.cell(x[None], s)[0][0]), s), cell=torch.nn.GRU(4, 16),
                                head=Lin(16, 3)),
        "lstm_sequence": _Module(lambda m, x, s: (m.head(m.cell(x[None], s)[0][0]), s), cell=torch.nn.LSTM(4, 16),
                                 head=Lin(16, 3)),
        "rnn_cell": _Module(_gru_head, cell=torch.nn.RNNCell(4, 16), head=Lin(16, 3)),
        "deeper_head": _Module(lambda m, x, s: (m.h2(torch.tanh(m.head(m.cell(x, s)))), m.cell(x, s)),
                               cell=G(4, 16), head=Lin(16, 16), h2=Lin(16, 3)),
        "linear_before_cell": _Module(lambda m, x, s: _gru_head(m, m.pre(x), s), pre=Lin(4, 4), cell=G(4, 16),
                                      head=Lin(16, 3)),
        "ignores_the_state": _Module(lambda m, x, s: _gru_head(m, x, None), cell=G(4, 16), head=Lin(16, 3)),
        "cell_without_bias": _Module(_gru_head, cell=G(4, 16, bias=False), head=Lin(16, 3)),
        "head_without_bias": _Module(_gru_head, cell=G(4, 16), head=Lin(16, 3, bias=False)),
        "head_registered_first": _Module(_gru_head, head=Lin(16, 3), cell=G(4, 16)),
        "sigmoid_output": _Module(lambda m, x, s: (torch.sigmoid(_gru_head(m, x, s)[0]), m.cell(x, s)),
                                  cell=G(4, 16), head=Lin(16, 3)),
        "lstm_returns_h_only": _Module(lambda m, x, s: (m.head(m.cell(x, s)[0]), m.cell(x, s)[0]), cell=L(4, 16),
                                       head=Lin(16, 3)),
        "mlp": _Module(lambda m, x, s: (m.head(torch.relu(m.l1(x))), s), l1=Lin(4, 16), head=Lin(16, 3)),
    }


@pytest.mark.parametrize("name", sorted(_non_forms()))
def test_rejects_every_non_form(name):
    torch.manual_seed(0)
    assert rnn_spec_from_module(_non_forms()[name]) is None


def test_recognition_leaves_the_global_rng_stream_untouched():
    torch.manual_seed(7)
    modules = [policy_class(c, t)(DIMS) for c in ("gru", "lstm") for t in (False, True)] + list(_non_forms().values())
    before = torch.get_rng_state()
    for m in modules:
        rnn_spec_from_module(m)
    assert torch.equal(before, torch.get_rng_state())


# ------------------------------------------------------------------ mode selection
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_population_mode_is_selected_for_a_recurrent_population_agent(cell):
    es = _es(cell=cell)
    assert es._fused and es._population and es._is_rnn and es._precision == "fp32"
    assert es.agent.device == es._dev
    es.train(n_steps=2)
    steps = es.agent.delay + 2
    assert es._be.act_calls == 2 * (steps + steps)        # population and centre episodes


class _OwnReturns(E.ES):
    def _calculate_returns(self, parameters):
        return super()._calculate_returns(parameters)


@pytest.mark.parametrize("case", ["sgd", "overridden_hook", "two_workers", "device_agent"])
def test_hooks_mode_serves_everything_else(case, monkeypatch):
    kw = {}
    if case == "sgd":
        kw["optimizer"] = torch.optim.SGD
    elif case == "overridden_hook":
        kw["cls"] = _OwnReturns
    elif case == "two_workers":
        monkeypatch.setenv("WORLD_SIZE", "2")
        monkeypatch.setenv("RANK", "0")
    if case == "device_agent":
        es = E.ES(policy_class("gru", True), DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
                  policy_kwargs={"dims": DIMS}, agent_kwargs={"obs": torch.zeros(2, 4), "target": torch.zeros(2, 3)},
                  noise_table_size=1 << 14, _backend=OracleBackend())
        assert es._is_rnn and not es._fused and not es._population
        return
    es = _es(**kw)
    assert es._is_rnn and not es._fused and not es._population
    assert es.agent.device == es.device
    if case != "two_workers":
        es.train(n_steps=1)
        assert es._be.act_calls == 0


def test_population_mode_refuses_a_tensor_core_precision():
    with pytest.raises(ValueError, match="fp32 only"):
        _es(eval_precision="f16")
    assert _es(eval_precision="fp32")._population


# ------------------------------------------------------------------ act
def _split(out, cell, H):
    y, s = out[..., :-state_width(cell, H)], out[..., -state_width(cell, H):]
    return y, (s if cell == "gru" else (s[..., :H], s[..., H:]))


@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_act_member_order_shapes_and_state(cell):
    P, H = 8, DIMS[1]
    es = _es(cell=cell, P=P)
    slot = es._slots[0]
    slot.theta_prev.copy_(slot.theta)
    es._draw_offsets()
    act = es._population_act(slot)
    rng = np.random.RandomState(0)
    S = state_width(cell, H)
    xs = rng.standard_normal((P, 3, 4 + S)).astype(np.float32)
    x = torch.from_numpy(xs[..., :4])
    st = torch.from_numpy(xs[..., 4:4 + H]) if cell == "gru" else \
        (torch.from_numpy(xs[..., 4:4 + H]), torch.from_numpy(xs[..., 4 + H:]))
    y, s = act(x, st)
    rows, _ = orc.sample_population(slot.theta.numpy(), es._table.numpy(), es._offsets.numpy(), es.sigma)
    want = step32(rows, cell, DIMS, xs, True)
    got = torch.cat([y, s] if cell == "gru" else [y, *s], -1).numpy()
    assert y.shape == (P, 3, 3) and (s.shape if cell == "gru" else s[1].shape) == (P, 3, H)
    np.testing.assert_array_equal(got, want)
    # row i < P/2 is theta + sigma*T[off_i], row P/2 + i its mirror, each on its own observations and state
    for m in (0, 3, 4, 7):
        pol = policy_class(cell, True)(DIMS)
        torch.nn.utils.vector_to_parameters(torch.from_numpy(rows[m]), pol.parameters())
        ym, sm = pol(x[m], st[m] if cell == "gru" else (st[0][m], st[1][m]))
        np.testing.assert_allclose(y[m].numpy(), ym.detach().numpy(), rtol=0, atol=2e-6)
        np.testing.assert_allclose(got[m, :, 3:], torch.cat([sm] if cell == "gru" else list(sm), -1).detach().numpy(),
                                   rtol=0, atol=2e-6)
    # [M, in] form, and state None = zeros
    y1, s1 = act(x[:, 0], None)
    zeros = torch.zeros(P, H) if cell == "gru" else (torch.zeros(P, H), torch.zeros(P, H))
    y0, s0 = act(x[:, 0], zeros)
    assert y1.shape == (P, 3)
    assert torch.equal(y1, y0) and (torch.equal(s1, s0) if cell == "gru" else
                                    torch.equal(s1[0], s0[0]) and torch.equal(s1[1], s0[1]))
    # the centre
    yc, sc = es._population_act(slot, centre=True)(x[:1, 0], None)
    wc = step32(slot.theta.numpy()[None], cell, DIMS, np.concatenate([xs[:1, :1, :4], np.zeros((1, 1, S), np.float32)],
                                                                     -1), True)
    np.testing.assert_array_equal(torch.cat([yc, sc] if cell == "gru" else [yc, *sc], -1).numpy(), wc[:, 0])
    with pytest.raises(ValueError, match="expected"):
        act(torch.zeros(7, 4))
    with pytest.raises(ValueError, match="state"):
        act(x, torch.zeros(P, 3, H + 1) if cell == "gru" else (torch.zeros(P, 3, H),))


def test_rollout_is_the_reference_protocol():
    ag = RecallAgent()
    for cell in ("gru", "lstm"):
        pol = policy_class(cell, True)(DIMS)
        r = ag.rollout(pol)
        assert isinstance(r, float)
        with torch.no_grad():
            ret = ag.rollout_population(lambda o, s: pol(o, s), 1)
        assert r == float(ret[0])
    r2, bc = RecallAgent(bc_dim=9).rollout(pol)
    assert isinstance(r2, float) and bc.shape == (9,)


def test_a_memoryless_policy_cannot_solve_the_recall_task():
    """The recall task needs memory: the best constant answer to the last observation scores MEMORYLESS_BEST."""
    ag = RecallAgent()
    target = 1.6 * torch.eye(3) - 0.8
    best = target.mean(0, keepdim=True).expand(3, 3)
    assert abs(float(-((best - target) ** 2).mean()) - RecallAgent.MEMORYLESS_BEST) < 1e-5
    # a perfect recurrent answer scores 0: feed the cue through the state by hand
    def act(o, s):
        s = o[..., :3] if s is None else s
        return (1.6 * s - 0.8), s
    assert float(ag.rollout_population(act, 2).max()) == 0.0


# ------------------------------------------------------------------ the reference goldens
class _Rec:
    def log(self):
        self.rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                             best=self.best_reward, idx=getattr(self, "idx", None),
                             archive=len(getattr(self, "_archive", []))))


def _load_theta(module, flat):
    torch.nn.utils.vector_to_parameters(torch.from_numpy(flat.copy()), module.parameters())


def run_es_golden(backend):
    """ES with the GRU policy in population mode from es_rnn_gru_p16.npz's start; returns (instance, fixture)."""
    g = load_golden("es_rnn_gru_p16.npz")

    class R(_Rec, E.ES):
        pass
    es = R(policy_class("gru", True), RecallAgent, torch.optim.Adam, population_size=16, sigma=float(g["sigma"]),
           policy_kwargs={"dims": tuple(int(d) for d in g["dims"])}, optimizer_kwargs={"lr": 0.01},
           noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]), _backend=backend)
    es.rec = []
    assert es._population and es._is_rnn
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
    """NSR-ES with the LSTM policy in population mode from nsr_rnn_lstm_p8.npz's start."""
    g = load_golden("nsr_rnn_lstm_p8.npz")

    class R(_Rec, E.NSR_ES):
        pass
    np.random.seed(123)
    es = R(policy_class("lstm", False), RecallAgent, torch.optim.Adam, population_size=8, sigma=float(g["sigma"]),
           policy_kwargs={"dims": tuple(int(d) for d in g["dims"])}, agent_kwargs={"bc_dim": 9},
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]),
           _backend=backend)
    es.rec = []
    assert es._population and es._is_rnn
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


def test_es_gru_population_mode_matches_reference_golden():
    check_es_golden(*run_es_golden(OracleBackend()))


def test_nsr_lstm_population_mode_matches_reference_golden():
    check_nsr_golden(*run_nsr_golden(OracleBackend()))


# ------------------------------------------------------------------ population mode against hooks mode
class _Hooks(E.ES):
    def _after_optimize(self, policy):          # any overridden hook selects hooks mode
        super()._after_optimize(policy)


@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_population_mode_matches_hooks_mode_on_the_same_agent(cell):
    runs = []
    for cls in (E.ES, _Hooks):
        torch.manual_seed(5)
        es = _es(cls=cls, cell=cell, P=8)
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
@pytest.mark.parametrize("cls,cell,bc_dim", [(E.ES, "gru", 0), (E.NSR_ES, "lstm", 9)])
def test_checkpoint_resume_is_bit_identical(cls, cell, bc_dim):
    torch.manual_seed(1)
    np.random.seed(1)
    a = _es(cls=cls, cell=cell, bc_dim=bc_dim)
    a.train(n_steps=3)
    torch.manual_seed(1)
    np.random.seed(1)
    b = _es(cls=cls, cell=cell, bc_dim=bc_dim)
    b.train(n_steps=2)
    sd = b.state_dict()
    torch.manual_seed(99)
    c = _es(cls=cls, cell=cell, bc_dim=bc_dim)
    c.load_state_dict(sd)
    c.train(n_steps=1)
    for sa, sc in zip(a._slots, c._slots):
        assert torch.equal(sa.theta, sc.theta) and torch.equal(sa.m, sc.m) and torch.equal(sa.v, sc.v)
    assert a.best_reward == c.best_reward
    np.testing.assert_array_equal(a.population_returns, c.population_returns)


# ------------------------------------------------------------------ ABI
def test_header_and_binding_agree_on_the_cell_codes():
    header = open(os.path.join(ROOT, "include", "estk.h")).read()
    for name, want in (("ESTK_CELL_GRU", CELL_GRU), ("ESTK_CELL_LSTM", CELL_LSTM)):
        m = re.search(r"#define\s+%s\s+(\d+)\b" % name, header)
        assert m and int(m.group(1)) == getattr(_capi, name) == want
    assert re.search(r"#define\s+ESTK_VERSION\s+200\b", header)
    for text in ("weight_ih", "weight_hh", "h' = fmaf(z, h - n, n)", "c' = fmaf(f, c, i*g)", "ESTK_CELL_GRU (8)",
                 "ESTK_CELL_LSTM (9)", "29 in all"):
        assert text in header, text


def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


CELL_CODES = [c | o | ACTIONS for c in (CELL_GRU, CELL_LSTM) for o in (0, 1 << 8)]
CELL_REFUSED = [c | rest for c in (CELL_GRU, CELL_LSTM) for rest in (0, 1 << 8, 1 << 16, 0x20000, 0x30200, 0x70000)]


def test_support_probe_refuses_the_cell_codes_under_every_precision():
    from estorch_b200.backend import mlp_desc
    lib = _lib()
    sup = lambda dims, code, prec, B: lib.estk_eval_mlp_supported(C.byref(mlp_desc(dims, code)), prec, B)  # noqa
    precs = (_capi.ESTK_PREC_FP32, _capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S,
             _capi.ESTK_PREC_F16_ANY)
    for code in CELL_CODES + CELL_REFUSED:
        for prec in precs:
            for dims in ([64, 64, 32], [64, 128, 64, 32]):
                assert sup(dims, code, prec, 256) == 0, (hex(code), prec, dims)
