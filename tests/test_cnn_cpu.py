"""Convolutional policies on fixed batches without a GPU: recognition (accepted forms and every excluded construct),
the global RNG left untouched, mode selection, fused mode against hooks mode on the oracle stand-in
(tests/_cnn_oracle.py), checkpoint / resume, and the CNN codes in the header, _capi and the library's support
probe."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch import nn

import estorch_b200.estorch as E
from estorch_b200 import DeviceAgent, PopulationAgent, SequenceAgent, _capi
from estorch_b200.policy_spec import CNNSpec, cnn_spec_from_module
from conftest import ROOT, load_golden, rel_err
from _cnn_oracle import CnnOracleBackend, forward, image_task, pack, param_count, policy_class, returns_of
from test_population_rnn_cpu import _load_theta, _Rec, check_es_golden, check_nsr_golden

SHAPE = (1, 12, 12)
DIMS = pack(SHAPE, [(4, 3, 2, 1), (6, 3, 2, 0)], [8, 4])


def _es(cls=E.ES, hidden="relu", out_tanh=False, optimizer=torch.optim.Adam, agent=DeviceAgent, agent_kwargs=None,
        P=8, dims=DIMS, loss="mse", **kw):
    obs, tgt = image_task(6, SHAPE, seed=2)
    if loss == "mse":
        tgt = tgt - 0.5
    es = cls(policy_class(2, hidden, out_tanh), agent, optimizer, population_size=P, sigma=0.05,
             policy_kwargs={"dims": dims}, agent_kwargs=agent_kwargs or dict(obs=obs, target=tgt, loss=loss),
             optimizer_kwargs={"lr": 0.02}, noise_table_size=1 << 13, _backend=CnnOracleBackend(), **kw)
    es.log = lambda: None
    return es


# ------------------------------------------------------------------ recognition
@pytest.mark.parametrize("form", ["sequential", "custom"])
@pytest.mark.parametrize("hidden", ["relu", "tanh", "elu", "silu", "leaky_relu"])
@pytest.mark.parametrize("out_tanh", [False, True])
def test_recognises_every_hidden_kind_and_output(form, hidden, out_tanh):
    torch.manual_seed(0)
    pol = policy_class(2, hidden, out_tanh, form)(DIMS)
    s = cnn_spec_from_module(pol, SHAPE)
    assert isinstance(s, CNNSpec) and s.dims == DIMS and s.hidden == hidden
    assert s.output == ("tanh" if out_tanh else "identity")
    assert s.act == {"relu": 0, "tanh": 1, "elu": 3, "silu": 4, "leaky_relu": 5}[hidden] | \
        (0x100 if out_tanh else 0) | 2 << 24
    assert s.n_parameters == param_count(DIMS, 2) == sum(p.numel() for p in pol.parameters())
    th = torch.nn.utils.parameters_to_vector(pol.parameters()).detach().numpy()
    x = torch.randn(3, *SHAPE)
    with torch.no_grad():
        assert np.abs(forward(th, DIMS, s.act, x.numpy(), np.float64) - pol(x).numpy()).max() < 1e-5


def test_valid_padding_and_view_forms():
    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.c = nn.Conv2d(3, 5, 3, padding="valid")
            self.f = nn.Linear(5 * 5 * 5, 2)

        def forward(self, x):
            return self.f(torch.relu(self.c(x)).view(x.shape[0], -1))
    s = cnn_spec_from_module(Net(), (3, 7, 7))
    assert s is not None and s.convs == ((5, 3, 1, 0),) and s.linears == (2,) and s.flat == 125


def _seq(*mods):
    return nn.Sequential(*mods)


NOT_CNNS = {
    "maxpool": lambda: _seq(nn.Conv2d(1, 4, 3), nn.ReLU(), nn.MaxPool2d(2), nn.Flatten(), nn.Linear(100, 2)),
    "batchnorm": lambda: _seq(nn.Conv2d(1, 4, 3), nn.BatchNorm2d(4), nn.ReLU(), nn.Flatten(), nn.Linear(400, 2)),
    "mixed_kinds": lambda: _seq(nn.Conv2d(1, 4, 3), nn.ReLU(), nn.Conv2d(4, 4, 3), nn.ELU(), nn.Flatten(),
                                nn.Linear(256, 2)),
    "conv_after_linear": lambda: _seq(nn.Linear(12, 12), nn.Unflatten(1, (1, 12)), nn.Conv2d(1, 2, 3)),
    "no_bias": lambda: _seq(nn.Conv2d(1, 4, 3, bias=False), nn.ReLU(), nn.Flatten(), nn.Linear(400, 2)),
    "groups": lambda: _seq(nn.Conv2d(2, 4, 3, groups=2), nn.ReLU(), nn.Flatten(), nn.Linear(400, 2)),
    "dilation": lambda: _seq(nn.Conv2d(1, 4, 3, dilation=2), nn.ReLU(), nn.Flatten(), nn.Linear(256, 2)),
    "rect_kernel": lambda: _seq(nn.Conv2d(1, 4, (3, 2)), nn.ReLU(), nn.Flatten(), nn.Linear(440, 2)),
    "rect_stride": lambda: _seq(nn.Conv2d(1, 4, 3, stride=(1, 2)), nn.ReLU(), nn.Flatten(), nn.Linear(200, 2)),
    "reflect_pad": lambda: _seq(nn.Conv2d(1, 4, 3, padding=1, padding_mode="reflect"), nn.ReLU(), nn.Flatten(),
                                nn.Linear(576, 2)),
    "same_pad": lambda: _seq(nn.Conv2d(1, 4, 3, padding="same"), nn.ReLU(), nn.Flatten(), nn.Linear(576, 2)),
    "no_linear": lambda: _seq(nn.Conv2d(1, 4, 3), nn.ReLU(), nn.Flatten()),
    "linear_no_bias": lambda: _seq(nn.Conv2d(1, 4, 3), nn.ReLU(), nn.Flatten(), nn.Linear(400, 2, bias=False)),
    "wrong_width": lambda: _seq(nn.Conv2d(1, 4, 3), nn.ReLU(), nn.Flatten(), nn.Linear(401, 2)),
    "elu_alpha": lambda: _seq(nn.Conv2d(1, 4, 3), nn.ELU(alpha=0.5), nn.Flatten(), nn.Linear(400, 2)),
    "dropout": lambda: _seq(nn.Conv2d(1, 4, 3), nn.ReLU(), nn.Dropout(), nn.Flatten(), nn.Linear(400, 2)),
}


@pytest.mark.parametrize("name", list(NOT_CNNS))
def test_excluded_constructs_return_none(name):
    torch.manual_seed(0)
    mod = NOT_CNNS[name]()
    shape = (2, 12, 12) if name == "groups" else (1, 12, 12)
    assert cnn_spec_from_module(mod, shape) is None


def test_vbn_policy_and_forward_that_differs_return_none():
    from _pop_conv_oracle import AtariPolicy          # the conv + VirtualBatchNorm policy of the Atari example
    pol = AtariPolicy(n_actions=4, xref=torch.rand(2, 4, 84, 84))
    assert cnn_spec_from_module(pol, (4, 84, 84)) is None

    class Doubled(nn.Module):
        def __init__(self):
            super().__init__()
            self.c, self.f = nn.Conv2d(1, 4, 3), nn.Linear(400, 2)

        def forward(self, x):
            return 2 * self.f(torch.relu(self.c(x)).flatten(1))
    assert cnn_spec_from_module(Doubled(), (1, 12, 12)) is None
    assert cnn_spec_from_module(policy_class(2)(DIMS), (1, 13, 12)) is None     # another frame size


def test_the_global_rng_is_untouched_and_existing_specs_unchanged():
    torch.manual_seed(7)
    want = torch.rand(5)
    pol = policy_class(2, "silu", True)(DIMS)
    torch.manual_seed(7)
    assert cnn_spec_from_module(pol, SHAPE) is not None
    assert torch.equal(torch.rand(5), want)
    # the ES constructor: an MLP policy is still an MLPSpec, a recurrent one an RNNSpec
    from test_api_cpu import MLP
    obs, tgt = torch.randn(6, 3), torch.randn(6, 2)
    es = E.ES(MLP, DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05, policy_kwargs={"dims": [3, 8, 2]},
              agent_kwargs=dict(obs=obs, target=tgt), noise_table_size=1 << 13, _backend=CnnOracleBackend())
    assert type(es._spec).__name__ == "MLPSpec" and not es._is_cnn
    # the conv + VirtualBatchNorm policy of the Atari example and a recurrent policy keep their specs
    from _pop_conv_oracle import AtariPolicy
    from _rnn_oracle import policy_class as rnn_policy_class
    from estorch_b200.policy_spec import ConvVBNSpec, RNNSpec
    from _pop_conv_oracle import PopConvOracleBackend
    # (SGD: hooks mode, so the stand-in needs no conv scratch; the spec is recognised the same way)
    es = E.ES(AtariPolicy, DeviceAgent, torch.optim.SGD, population_size=8, sigma=0.05,
              policy_kwargs={"n_actions": 4, "xref": torch.rand(3, 4, 84, 84)}, optimizer_kwargs={"lr": 0.01},
              agent_kwargs=dict(obs=torch.rand(2, 4, 84, 84), target=torch.rand(2, 4)), noise_table_size=1 << 20,
              _backend=PopConvOracleBackend())
    assert isinstance(es._spec, ConvVBNSpec) and es._spec.n_actions == 4 and not es._is_cnn
    g = torch.Generator().manual_seed(9)
    es = E.ES(rnn_policy_class("lstm", True), SequenceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
              policy_kwargs={"dims": (3, 8, 2)},
              agent_kwargs=dict(obs=torch.randn(5, 4, 3, generator=g), target=torch.rand(5, 4, 2, generator=g)),
              noise_table_size=1 << 13, _backend=CnnOracleBackend())
    assert es._spec == RNNSpec("lstm", (3, 8, 2), "tanh") and not es._is_cnn


# ------------------------------------------------------------------ mode selection
@pytest.mark.parametrize("loss", ["mse", "cross_entropy"])
def test_fused_mode_is_selected_for_a_cnn_on_a_device_agent(loss):
    es = _es(loss=loss)
    assert es._fused and es._is_cnn and not es._population and es._precision == "fp32"
    assert es._act_code() == 2 << 24 | (_capi.ESTK_LOSS_XENT if loss == "cross_entropy" else 0)
    ns = _es(cls=E.NSR_ES, agent_kwargs=dict(obs=image_task(6, SHAPE)[0], target=image_task(6, SHAPE)[1],
                                             bc_obs=2, bc_dim=8))
    assert ns._fused and ns._is_cnn


class _Hooks(E.ES):
    def _after_optimize(self, policy):          # any overridden hook selects hooks mode
        super()._after_optimize(policy)


class _Pop(PopulationAgent):
    def __init__(self, **_):
        pass

    def rollout_population(self, act, members):
        return np.zeros(members, np.float32)


@pytest.mark.parametrize("case", ["sgd", "hook", "k", "population", "sequence", "shape", "xent_tanh"])
def test_hooks_mode_serves_everything_else(case):
    obs, tgt = image_task(6, SHAPE, seed=2)
    if case == "sgd":
        es = _es(optimizer=torch.optim.SGD)
    elif case == "hook":
        es = _es(cls=_Hooks)
    elif case == "k":
        es = _es(cls=E.NS_ES, k=33, agent_kwargs=dict(obs=obs, target=tgt, bc_obs=1, bc_dim=4))
    elif case == "population":
        es = _es(agent=_Pop, agent_kwargs={})
    elif case == "sequence":
        es = _es(agent=SequenceAgent, agent_kwargs=dict(obs=obs.reshape(6, 12, 12), target=tgt[:, None].expand(6, 12, 4)))
    elif case == "shape":
        es = _es(agent_kwargs=dict(obs=torch.randn(6, 1, 13, 13), target=tgt))
    else:
        es = _es(out_tanh=True, loss="cross_entropy")
    assert not es._fused and not es._population


def test_fused_mode_refuses_a_tensor_core_precision():
    for prec in ("f16", "bf16", "bf16s"):
        with pytest.raises(ValueError, match="fp32 only"):
            _es(eval_precision=prec)
    assert _es(eval_precision="fp32")._fused


# ------------------------------------------------------------------ the reference goldens
def run_es_cnn_golden(backend):
    """ES with the ReLU / Tanh-output CNN in fused mode from es_cnn_p16.npz's start; returns (instance, fixture)."""
    g = load_golden("es_cnn_p16.npz")

    class R(_Rec, E.ES):
        pass
    es = R(policy_class(2, "relu", True), DeviceAgent, torch.optim.Adam, population_size=16, sigma=float(g["sigma"]),
           policy_kwargs={"dims": tuple(int(d) for d in g["dims"])}, optimizer_kwargs={"lr": 0.01},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"])),
           noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]), _backend=backend)
    es.rec = []
    assert es._fused and es._is_cnn and es._spec.output == "tanh"
    es._table.copy_(torch.from_numpy(g["table"]).to(es._dev))
    _load_theta(es.policy, g["theta0"])
    es._slots[0].ensure_flat()
    es.train(n_steps=3)
    return es, g


def run_nsr_cnn_golden(backend):
    """NSR-ES with the Tanh-hidden CNN, cross-entropy and an 8-D BC, from nsr_cnn_xent_p8.npz's start."""
    g = load_golden("nsr_cnn_xent_p8.npz")

    class R(_Rec, E.NSR_ES):
        pass
    np.random.seed(123)
    es = R(policy_class(2, "tanh", False), DeviceAgent, torch.optim.Adam, population_size=8, sigma=float(g["sigma"]),
           policy_kwargs={"dims": tuple(int(d) for d in g["dims"])}, optimizer_kwargs={"lr": 0.01},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]),
                             bc_obs=int(g["bc_obs"]), bc_dim=int(g["bc_dim"]), loss="cross_entropy"),
           noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]), _backend=backend)
    es.rec = []
    assert es._fused and es._is_cnn and es._spec.hidden == "tanh"
    es._table.copy_(torch.from_numpy(g["table"]).to(es._dev))
    for i, (p, _) in enumerate(es.meta_population):
        _load_theta(p, g["meta_theta0"][i])
        es._slots[i].ensure_flat()
        es._slots[i].push_theta()
    es._archive = [a.copy() for a in g["archive0"]]
    np.random.seed(123)
    es.train(n_steps=len(g["grad"]))
    return es, g


def test_es_cnn_matches_reference_golden():
    check_es_golden(*run_es_cnn_golden(CnnOracleBackend()))


def test_nsr_cnn_cross_entropy_matches_reference_golden():
    check_nsr_golden(*run_nsr_cnn_golden(CnnOracleBackend()))


# ------------------------------------------------------------------ two processes over gloo
def test_world2_equals_world1(tmp_path):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="1")
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "_cnn_dist_worker.py"),
                                       str(tmp_path)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
    outs = [p.communicate(timeout=600)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o[-3000:]
    r0, r1 = (np.load(os.path.join(tmp_path, f"rank{r}.npz")) for r in range(2))
    assert int(r0["world"]) == 2 and int(r0["pairs_local"]) == 4 and int(r0["cnn_calls"]) > 0
    for k in ("theta", "returns", "episode"):
        np.testing.assert_array_equal(r0[k], r1[k])
    from _cnn_dist_worker import run
    es, _ = run()
    assert es.n_workers == 1
    assert rel_err(r0["returns"][:, 0], es.population_returns[:, 0]) < 1e-5
    assert rel_err(r0["theta"], es._slots[0].theta.numpy()) < 1e-5


# ------------------------------------------------------------------ fused against hooks mode, launches, resume
@pytest.mark.parametrize("cls,loss", [(E.ES, "mse"), (E.ES, "cross_entropy"), (E.NSR_ES, "cross_entropy")])
def test_fused_mode_matches_hooks_mode(cls, loss):
    runs = []
    obs, tgt = image_task(6, SHAPE, seed=2)
    kw = dict(obs=obs, target=tgt, loss=loss) if cls is E.ES else dict(obs=obs, target=tgt, loss=loss, bc_obs=2,
                                                                       bc_dim=8)
    hooks_cls = _Hooks if cls is E.ES else type("H", (cls,), {"_after_optimize": lambda s, p: cls._after_optimize(s, p)})
    for c in (cls, hooks_cls):
        torch.manual_seed(5)
        np.random.seed(5)
        es = _es(cls=c, agent_kwargs=kw)
        rec = []
        es.log = lambda es=es, rec=rec: rec.append((es.population_returns.copy(), es.episode_reward))
        es.train(n_steps=3)
        mods = [es.policy] if cls is E.ES else [p for p, _ in es.meta_population]
        theta = np.concatenate([torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy() for m in mods])
        runs.append((es._fused, rec, theta))
    (fused, f_rec, f_theta), (hooks, h_rec, h_theta) = runs
    assert fused and not hooks
    for (rf, ef), (rh, eh) in zip(f_rec, h_rec):
        assert rel_err(rf[:, 0], rh[:, 0]) < 1e-5
        assert abs(ef - eh) < 1e-5 * abs(eh)
    assert rel_err(f_theta, h_theta) < 2e-4


def test_one_population_and_one_centre_evaluate_per_generation():
    es = _es()
    es.train(n_steps=3)
    assert es._be.cnn_calls == 2 * 3


@pytest.mark.parametrize("cls,bc", [(E.ES, False), (E.NSR_ES, True)])
def test_checkpoint_resume_is_bit_identical(cls, bc):
    obs, tgt = image_task(6, SHAPE, seed=2)
    kw = dict(obs=obs, target=tgt, bc_obs=2, bc_dim=8) if bc else None

    def make(seed):
        torch.manual_seed(seed)
        return _es(cls=cls, agent_kwargs=kw)
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
    assert a.best_reward == c.best_reward
    np.testing.assert_array_equal(a.population_returns, c.population_returns)


def test_the_stand_in_evaluate_is_the_oracle_forward():
    es = _es(P=8)
    slot = es._slots[0]
    es._draw_offsets()
    ret = torch.zeros(8)
    es._be.eval_cnn(DIMS, slot.theta, es._table, es._offsets, es._order, 4, es.sigma, es._obs, es._tgt,
                    ret[:4], ret[4:], act=es._act_code())
    from oracle import es_oracle as orc
    rows, _ = orc.sample_population(slot.theta.numpy(), es._table.numpy(), es._offsets.numpy(), es.sigma)
    y = np.stack([forward(r, DIMS, es._act_code(), es._obs.numpy()) for r in rows])
    np.testing.assert_array_equal(ret.numpy(), returns_of(y, es._tgt.numpy(), False))


# ------------------------------------------------------------------ ABI
def test_header_and_capi_document_the_cnn_codes():
    header = open(os.path.join(ROOT, "include", "estk.h")).read()
    for text in ("Convolutional evaluate (bits 24-31 = n_conv", "ESTK_CNN_INPUT(c, h, w)",
                 "ESTK_CNN_CONV(out_c, k, stride, pad)", "ascending (ci, kh, kw) order", "-(S / (float)(B*out))",
                 "-(S / (float)B)", "the bits of the fp32\n * MLP evaluate's first Linear",
                 "#define ESTK_CNN_INPUT(c, h, w) ((int32_t)((uint32_t)(c) | (uint32_t)(h) << 10 | (uint32_t)(w) << 20))",
                 "(uint32_t)(out_c) | (uint32_t)(k) << 12 | (uint32_t)(stride) << 18 | (uint32_t)(pad) << 24"):
        assert text in header, text
    assert _capi.ESTK_CNN_INPUT(3, 5, 7) == 3 | 5 << 10 | 7 << 20
    assert _capi.ESTK_CNN_CONV(16, 8, 4, 2) == 16 | 8 << 12 | 4 << 18 | 2 << 24
    assert _capi.ESTK_CNN_N_CONV(3) == 3 << 24 and _capi.ESTK_CNN_MAX_CONV == 7
    assert _capi.ESTK_CNN_INPUT(*SHAPE) == DIMS[0] and _capi.ESTK_CNN_CONV(4, 3, 2, 1) == DIMS[1]


def test_support_probe_returns_0_for_cnn_codes():
    from estorch_b200.backend import cnn_desc
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = _capi.load()
    for n_conv in (1, 2, 7):
        for low in (0, 1, 0x100, _capi.ESTK_LOSS_XENT, 5 | 0x100):
            dims = pack((64, 1, 1), [(64, 1, 1, 0)] * n_conv, [32] if n_conv == 7 else [64, 32])
            for prec in range(5):
                d = cnn_desc(dims, low | n_conv << 24)
                assert lib.estk_eval_mlp_supported(C.byref(d), prec, 256) == 0, (n_conv, hex(low), prec)
