"""The TF32 convolutional evaluate without a GPU: the companion header and its binding, refusals through the ABI
before any launch (fake device pointers: nothing is dereferenced), the engine's eval_precision="tf32" mode
selection on the TF32 stand-in backend (tests/_cnn_tf32_oracle.py), and the numpy restatement of rna_tf32."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import estorch_b200.estorch as E
from estorch_b200 import DeviceAgent, PopulationAgent, _capi
from estorch_b200.backend import cnn_desc
from conftest import ROOT
from _cnn_oracle import image_task, pack, policy_class
from _batch_oracle import BatchMixin
from _cnn_tf32_oracle import LOSS_ACCURACY, Tf32CnnOracleBackend, rna_tf32

SHAPE = (1, 12, 12)
DIMS = pack(SHAPE, [(4, 3, 2, 1), (6, 3, 2, 0)], [8, 4])
HEADER = os.path.join(ROOT, "include", "estk_eval_cnn_tf32.h")
LIB = os.path.join(ROOT, "estorch_b200", "lib", "libestk.so")
needs_lib = pytest.mark.skipif(not os.path.exists(LIB), reason="libestk.so not built")


def _es(cls=E.ES, loss="mse", backend=None, agent_kwargs=None, P=8, **kw):
    obs, tgt = image_task(6, SHAPE, seed=2)
    if loss == "mse":
        tgt = tgt - 0.5
    es = cls(policy_class(2), DeviceAgent, torch.optim.Adam, population_size=P, sigma=0.05,
             policy_kwargs={"dims": DIMS}, agent_kwargs=agent_kwargs or dict(obs=obs, target=tgt, loss=loss),
             optimizer_kwargs={"lr": 0.02}, noise_table_size=1 << 13,
             _backend=backend or Tf32CnnOracleBackend(), **kw)
    es.log = lambda: None
    return es


# ------------------------------------------------------------------ header and binding
def _declared(path):
    src = open(path).read()
    return {m.group(1): m.group(2) for m in re.finditer(r"ESTK_API\s+[\w\s*]+?\b(estk_\w+)\s*\(([^;]*)\);", src)}


def test_header_declares_exactly_the_two_entry_points():
    src = open(HEADER).read()
    assert '#include "estk.h"' in src
    decl = _declared(HEADER)
    assert set(decl) == {"estk_eval_cnn_tf32", "estk_eval_cnn_tf32_supported"}
    assert set(decl) == set(_capi.EVAL_CNN_TF32_SIGNATURES)
    for name, args in decl.items():
        assert len(args.split(",")) == len(_capi.EVAL_CNN_TF32_SIGNATURES[name]), name
    for table in (_capi.SIGNATURES, _capi.BATCH_SIGNATURES, _capi.ACT_CNN_SIGNATURES):
        assert not set(decl) & set(table)


def test_core_header_is_unchanged():
    core = os.path.join(ROOT, "include", "estk.h")
    src = open(core).read()
    assert len(_declared(core)) == 25
    assert re.search(r"#define ESTK_VERSION 200\b", src)
    assert "TF32" not in "".join(re.findall(r"#define (ESTK_PREC_\w+)", src))


# ------------------------------------------------------------------ refusals through the ABI
FAKE = C.c_void_p(256)


def _desc(code, dims=DIMS):
    d = _capi.EstkMlpDesc()
    d.n_layers = len(dims) - 1
    for i, w in enumerate(dims):
        d.dims[i] = C.c_int32(int(w)).value
    d.activation = C.c_int32(int(code)).value
    return d


def _call(lib, d, ctx=FAKE, theta=FAKE, obs=FAKE, target=FAKE, rp=FAKE, rm=FAKE, B=6, pairs=4, table=FAKE,
          offsets=FAKE, bcp=None, bcm=None, bc_obs=0, bc_dim=0):
    return lib.estk_eval_cnn_tf32(ctx, C.byref(d) if d is not None else None, theta, table, offsets, None, pairs,
                                  0.05, obs, target, B, rp, rm, bcp, bcm, bc_obs, bc_dim, None)


GOOD = 2 << 24 | _capi.ESTK_LOSS_XENT
REFUSED = {
    "null ctx": dict(ctx=None), "null desc": dict(d=None), "null theta": dict(theta=None), "null obs": dict(obs=None),
    "null target": dict(target=None), "null ret_plus": dict(rp=None), "null ret_minus": dict(rm=None),
    "null table": dict(table=None), "B 0": dict(B=0), "pairs 0": dict(pairs=0),
    "pairs too many": dict(pairs=_capi.ESTK_MAX_POPULATION // 2 + 1), "bc one sided": dict(bcp=FAKE, bc_obs=1, bc_dim=1),
    "bc dims": dict(bcp=FAKE, bcm=FAKE), "n_conv 0": dict(code=0), "n_conv 8": dict(code=8 << 24),
    "actions": dict(code=2 << 24 | _capi.ESTK_ACTIONS), "gru cell": dict(code=2 << 24 | _capi.ESTK_CELL_GRU),
    "lstm cell": dict(code=2 << 24 | _capi.ESTK_CELL_LSTM), "loss value 2": dict(code=2 << 24 | 2 << 16),
    "xent with tanh": dict(code=GOOD | _capi.ESTK_ACT_OUT_TANH), "hidden 2": dict(code=2 << 24 | 2),
    "pad >= k": dict(dims=pack(SHAPE, [(4, 3, 2, 3), (6, 3, 2, 0)], [8, 4])),
    "zero channels": dict(dims=pack(SHAPE, [(0, 3, 2, 1), (6, 3, 2, 0)], [8, 4])),
    "conv larger than input": dict(dims=pack(SHAPE, [(4, 13, 1, 0), (6, 3, 2, 0)], [8, 4])),
    "no linear": dict(dims=pack(SHAPE, [(4, 3, 2, 1), (6, 3, 2, 0)], [])),
    "zero width": dict(dims=pack(SHAPE, [(4, 3, 2, 1), (6, 3, 2, 0)], [0, 4])),
}


@needs_lib
@pytest.mark.parametrize("case", list(REFUSED))
def test_refusals_before_any_launch(case):
    lib = _capi.load()
    kw = dict(REFUSED[case])
    code, dims = kw.pop("code", GOOD), kw.pop("dims", DIMS)
    d = kw.pop("d", _desc(code, dims))
    assert _call(lib, d, **kw) == -1, lib.estk_last_error()
    if d is not None and "B" not in kw:
        sup = lib.estk_eval_cnn_tf32_supported(C.byref(d), 6)
        assert sup == (0 if ("code" in REFUSED[case] or "dims" in REFUSED[case]) else 1), case
    if "B" in kw:
        assert lib.estk_eval_cnn_tf32_supported(C.byref(_desc(GOOD)), 0) == 0


@needs_lib
def test_supported_takes_every_return_code_and_the_required_shapes():
    lib = _capi.load()
    shapes = [((1, 28, 28), [(16, 5, 2, 2), (32, 5, 2, 2)], [10]), ((4, 84, 84), [(16, 8, 4, 0), (32, 4, 2, 0)],
              [256, 6]), ((6, 10, 10), [(16, 3, 1, 0)], [128, 4]), ((3, 128, 128), [(32, 3, 1, 1), (4, 8, 8, 0)], [4]),
              ((2, 13, 13), [(3, 3, 2, 2), (7, 3, 1, 0), (5, 1, 1, 0), (4, 3, 1, 1)], [9, 6, 2]),
              ((1, 28, 28), [(16, 5, 2, 2), (32, 5, 2, 2)], [64, 10])]
    for shape, convs, linears in shapes:
        for h in (0, 1, 3, 4, 5):
            for rest in (0, _capi.ESTK_ACT_OUT_TANH, _capi.ESTK_LOSS_XENT, LOSS_ACCURACY):
                d = cnn_desc(pack(shape, convs, linears), len(convs) << 24 | h | rest)
                for B in (1, 7, 256):
                    assert lib.estk_eval_cnn_tf32_supported(C.byref(d), B) == 1, (shape, h, rest, B)
    # a layer output beyond 2^26 floats per image is valid for the fp32 route and not served here
    d = cnn_desc(pack((1, 1023, 1023), [(100, 1, 1, 0)], [2]), 1 << 24)
    assert lib.estk_eval_cnn_tf32_supported(C.byref(d), 1) == 0
    rc = _call(lib, d, B=1)
    assert rc == _capi_unsupported(), lib.estk_last_error()


def _capi_unsupported():
    src = open(os.path.join(ROOT, "include", "estk.h")).read()
    return int(re.search(r"ESTK_ERR_UNSUPPORTED\s*=\s*(-?\d+)", src).group(1))


# ------------------------------------------------------------------ engine mode selection
@pytest.mark.parametrize("loss", ["mse", "cross_entropy", "accuracy"])
def test_tf32_is_fused_for_a_cnn_with_every_loss(loss):
    es = _es(loss=loss, eval_precision="tf32")
    assert es._fused and es._is_cnn and es._precision == "tf32"
    es.train(n_steps=2)
    assert set(es._be.cnn_precisions) == {"tf32"} and len(es._be.cnn_precisions) == 4


def test_auto_stays_fp32():
    es = _es(eval_precision="auto")
    assert es._precision == "fp32"
    es.train(n_steps=1)
    assert set(es._be.cnn_precisions) == {"fp32"}


def test_tf32_with_batch_size_and_nsr_with_bc():
    obs, tgt = image_task(40, SHAPE, seed=2)
    class Sampling(BatchMixin, Tf32CnnOracleBackend):
        pass
    es = _es(agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy", batch_size=8), eval_precision="tf32",
             backend=Sampling())
    assert es._fused and es._precision == "tf32"
    es.train(n_steps=2)
    assert set(es._be.cnn_precisions) == {"tf32"}
    es = _es(cls=E.NSR_ES, agent_kwargs=dict(obs=obs[:6], target=tgt[:6], loss="cross_entropy", bc_obs=2, bc_dim=8),
             eval_precision="tf32")
    assert es._fused and es._precision == "tf32"
    es.train(n_steps=2)
    assert set(es._be.cnn_precisions) == {"tf32"}


def test_refusals_in_the_engine():
    for prec in ("f16", "bf16", "bf16s"):
        with pytest.raises(ValueError, match="fp32 only"):
            _es(eval_precision=prec)
    with pytest.raises(ValueError, match="2\\*\\*26 floats"):
        _es(eval_precision="tf32", backend=Tf32CnnOracleBackend(tf32_supported=False))
    with pytest.raises(ValueError, match="'tf32'"):
        _es(eval_precision="tf33")
    # an MLP on a device agent
    from _oracle_backend import OracleBackend
    from estorch_b200.policy_spec import MLPSpec  # noqa: F401

    class MLP(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.l1, self.a, self.l2 = torch.nn.Linear(4, 8), torch.nn.ReLU(), torch.nn.Linear(8, 2)

        def forward(self, x):
            return self.l2(self.a(self.l1(x)))
    g = torch.Generator().manual_seed(0)
    with pytest.raises(ValueError, match="'tf32' is for convolutional policies"):
        E.ES(MLP, DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
             agent_kwargs=dict(obs=torch.randn(6, 4, generator=g), target=torch.randn(6, 2, generator=g)),
             noise_table_size=1 << 13, eval_precision="tf32", _backend=OracleBackend())


def test_a_fused_recurrent_policy_refuses_tf32():
    from estorch_b200 import SequenceAgent
    from _cnn_oracle import CnnOracleBackend
    from _rnn_oracle import policy_class as rnn_policy_class
    g = torch.Generator().manual_seed(9)
    kw = dict(policy_kwargs={"dims": (3, 8, 2)},
              agent_kwargs=dict(obs=torch.randn(5, 4, 3, generator=g), target=torch.rand(5, 4, 2, generator=g)),
              noise_table_size=1 << 13, _backend=CnnOracleBackend())
    es = E.ES(rnn_policy_class("lstm", True), SequenceAgent, torch.optim.Adam, population_size=8, sigma=0.05, **kw)
    assert es._fused and es._is_rnn
    with pytest.raises(ValueError, match="'tf32' is for convolutional policies"):
        E.ES(rnn_policy_class("lstm", True), SequenceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
             eval_precision="tf32", **kw)


def test_population_mode_refuses_tf32():
    class Pop(PopulationAgent):
        obs_shape = SHAPE

        def rollout_population(self, act, n):   # never reached
            raise AssertionError
    with pytest.raises(ValueError, match="fp32 only"):
        E.ES(policy_class(2), Pop, torch.optim.Adam, population_size=8, sigma=0.05, policy_kwargs={"dims": DIMS},
             noise_table_size=1 << 13, eval_precision="tf32", _backend=Tf32CnnOracleBackend())


def test_hooks_mode_ignores_tf32():
    class Hooks(E.ES):
        def _after_optimize(self, policy):
            super()._after_optimize(policy)
    es = _es(cls=Hooks, eval_precision="tf32")
    assert not es._fused and es._precision == "fp32"


def test_resume_continues_bit_for_bit():
    def make(seed):
        torch.manual_seed(seed)
        return _es(eval_precision="tf32")
    np.random.seed(1)
    a = make(1)
    a.train(n_steps=3)
    np.random.seed(1)
    b = make(1)
    b.train(n_steps=2)
    sd = b.state_dict()
    c = make(99)
    c.load_state_dict(sd)
    c.train(n_steps=1)
    for sa, sc in zip(a._slots, c._slots):
        assert torch.equal(sa.theta, sc.theta) and torch.equal(sa.m, sc.m) and torch.equal(sa.v, sc.v)
    np.testing.assert_array_equal(a.population_returns, c.population_returns)


# ------------------------------------------------------------------ rna_tf32 restatement
def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def test_rna_tf32_rounds_ties_away_from_zero_on_both_signs():
    one = np.float32(1.0)
    tie = np.float32(1 + 2.0 ** -11)          # halfway between 1 and 1 + 2^-10
    assert rna_tf32(tie) == np.float32(1 + 2.0 ** -10)
    assert rna_tf32(-tie) == -np.float32(1 + 2.0 ** -10)
    below = np.nextafter(tie, one)
    assert rna_tf32(below) == one and rna_tf32(-below) == -one
    assert rna_tf32(np.float32(1 + 3 * 2.0 ** -11)) == np.float32(1 + 2.0 ** -9)   # an odd tie goes up too
    x = np.random.RandomState(0).standard_normal(10000).astype(np.float32)
    r = rna_tf32(x)
    assert (_bits(r) & 0x1FFF == 0).all()
    assert (np.abs(r.astype(np.float64) - x) <= np.abs(x.astype(np.float64)) * 2.0 ** -11).all()
    assert np.array_equal(np.sign(r), np.sign(x))


def test_rna_tf32_special_values():
    big = np.float32(np.finfo(np.float32).max)
    assert np.isinf(rna_tf32(big)) and rna_tf32(big) > 0 and np.isinf(rna_tf32(-big))
    just_below = np.float32(np.frombuffer(np.uint32(0x7F7FEFFF).tobytes(), np.float32)[0])
    assert np.isfinite(rna_tf32(just_below)) and _bits(rna_tf32(just_below)) == 0x7F7FE000
    assert np.isnan(rna_tf32(np.float32(np.nan)))
    payload = np.frombuffer(np.uint32(0x7F800001).tobytes(), np.float32)
    assert np.isnan(rna_tf32(payload)).all()
    assert _bits(rna_tf32(np.float32(0.0))) == 0 and _bits(rna_tf32(np.float32(-0.0))) == 0x80000000
    assert np.isinf(rna_tf32(np.float32(np.inf))) and rna_tf32(np.float32(-np.inf)) < 0
