"""Classification accuracy as the return, without a GPU: ``DeviceAgent(loss="accuracy")``, the ESTK_LOSS_ACCURACY
code of ``estk_mlp_desc.activation`` in the header, the binding and the library's shape query, the fused / hooks
decision and the precision it picks, the tie and NaN rule of the restated return against ``torch.argmax``, and ES /
NSR-ES through the oracle stand-in (tests/_oracle_backend.py) against the reference-generated goldens."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
import _mlp_oracle as mlp
from _mlp_oracle import MLP
from _oracle_backend import OracleBackend
from _cnn_oracle import image_task, pack, policy_class as cnn_policy_class
import estorch_b200 as E
from estorch_b200 import _capi
from estorch_b200.batches import batch_indices

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ the return
def test_the_cpu_mean_of_a_count_is_one_ieee_divide():
    """The restated return (count / B in fp32) is what torch's CPU mean of the 0 / 1 rows gives, for every count."""
    for B in (1, 2, 3, 7, 10, 100, 255, 256, 257, 1000, 60000):
        counts = np.unique(np.linspace(0, B, min(B + 1, 400)).astype(np.int64))
        for c in counts:
            rows = torch.zeros(B)
            rows[:c] = 1.0
            want = np.float32(np.float32(c) / np.float32(B))
            assert np.float32(rows.mean()) == want, (B, c)
            assert np.float32(rows.mean()).tobytes() == want.tobytes()


def test_ties_and_nans_follow_torch_argmax():
    y = torch.tensor([[1.0, 3.0, 3.0, 0.0],           # a tie: the lower index
                      [2.0, float("nan"), 5.0, float("nan")],   # the first NaN wins over a larger number
                      [-float("inf")] * 4,              # all -inf: index 0
                      [0.0, -0.0, 0.0, -1.0],           # -0 == +0: index 0
                      [float("nan")] * 4,
                      [1.0, 2.0, float("inf"), float("inf")],
                      [-1.0, -1.0, -2.0, -1.0]])
    t = F.one_hot(torch.tensor([1, 1, 0, 0, 0, 2, 0]), 4).float()
    assert np.array_equal(np.argmax(y.numpy(), 1), y.argmax(1).numpy())
    assert np.array_equal(mlp.correct_rows(y.numpy(), t.numpy()), (y.argmax(1) == t.argmax(1)).numpy())
    assert mlp.correct_rows(y.numpy(), t.numpy()).tolist() == [True, True, True, True, True, True, True]
    soft = torch.tensor([[0.25, 0.25, 0.5, 0.0]] * 7)  # a soft target's label is its first largest weight
    assert mlp.accuracy_return(y.numpy(), soft.numpy()) == np.float32(np.float32(1) / np.float32(7))   # row 5 only
    pol = torch.nn.Identity()
    pol.register_parameter("p", torch.nn.Parameter(torch.zeros(1)))
    for tgt in (t, soft):
        r = E.DeviceAgent(torch.zeros(7, 4), tgt, loss="accuracy")
        r.obs = y                                     # the logits themselves through an identity policy
        assert r.rollout(pol) == float(mlp.accuracy_return(y.numpy(), tgt.numpy()))


def test_rollout_is_the_fraction_of_correct_rows_and_bc_the_logits():
    g = torch.Generator().manual_seed(0)
    pol = MLP([6, 16, 5], "relu")
    obs = torch.randn(50, 6, generator=g)
    labels = torch.randint(0, 5, (50,), generator=g)
    r, bc = E.DeviceAgent(obs, F.one_hot(labels, 5).float(), bc_obs=4, bc_dim=18, loss="accuracy").rollout(pol)
    with torch.no_grad():
        out = pol(obs)
    assert r == float((out.argmax(1) == labels).float().mean())
    np.testing.assert_array_equal(bc, out[:4].flatten()[:18].numpy())


@pytest.mark.parametrize("target", [
    -torch.ones(4, 3),
    torch.tensor([[0.5, float("nan"), 0.5]] * 4),
    torch.tensor([[0.0, float("inf"), 0.0]] * 4),
    torch.ones(4, 3, dtype=torch.int64),
])
def test_bad_targets_raise(target):
    with pytest.raises(ValueError, match="accuracy"):
        E.DeviceAgent(torch.randn(4, 2), target, loss="accuracy")


def test_a_batch_of_2_24_rows_is_refused_before_it_is_copied():
    big = torch.zeros(1, 1).expand(1 << 24, 1)           # no storage behind the rows
    with pytest.raises(ValueError, match="2\\^24"):
        E.DeviceAgent(big, big, loss="accuracy")
    with pytest.raises(ValueError, match="2\\^24"):
        E.DeviceAgent(big, big, loss="accuracy", batch_size=1 << 24)
    assert E.DeviceAgent(torch.zeros(10, 1), torch.ones(10, 2), loss="accuracy", batch_size=4).batch_size == 4


def test_sequence_agent_refuses_the_accuracy():
    with pytest.raises(ValueError, match="SequenceAgent"):
        E.SequenceAgent(torch.randn(4, 3, 2), torch.ones(4, 3, 2), loss="accuracy")


# ------------------------------------------------------------------ the code in the header, binding and library
def test_header_and_binding_agree():
    header = open(os.path.join(ROOT, "include", "estk.h")).read()
    m = re.search(r"#define\s+ESTK_LOSS_ACCURACY\s+\((\d+) << 16\)", header)
    assert m and int(m.group(1)) << 16 == _capi.ESTK_LOSS_ACCURACY == mlp.LOSS_ACCURACY == 0x60000
    assert _capi.ESTK_LOSS_ACCURACY & _capi.ESTK_LOSS_XENT == 0     # bit 16 clear: never read as the cross-entropy
    assert re.search(r"#define\s+ESTK_VERSION\s+200\b", header)


def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


def _supported(lib, dims, act, precision, B=256):
    from estorch_b200.backend import mlp_desc
    return lib.estk_eval_mlp_supported(C.byref(mlp_desc(dims, act)), precision, B)


def test_supported_query_follows_the_cross_entropy():
    lib = _lib()
    north = [128, 512, 512, 512, 512, 256]
    TC = (_capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S, _capi.ESTK_PREC_F16_ANY)
    for h in (0, 1, 3, 4, 5):
        for prec in TC:
            for dims, B in ((north, 256), ([64, 64, 32], 256), ([784, 256, 10], 100), (north, 100)):
                assert _supported(lib, dims, h | 0x60000, prec, B) == _supported(lib, dims, h | 0x10000, prec, B), \
                    (h, prec, dims, B)
        assert _supported(lib, north, h | 0x60000, _capi.ESTK_PREC_F16) == 1
        assert _supported(lib, north, h | 0x60000, _capi.ESTK_PREC_FP32) == 0   # not a tensor-core precision
    for code in (0x60100, 0x60101, 0x60008, 0x60009, 0x70000, 0x60002, 0x60000 | 3 << 16):
        for prec in TC:
            assert _supported(lib, north, code, prec) == 0, (hex(code), prec)


# ------------------------------------------------------------------ fused or hooks, and the precision
def _es(hidden="relu", output="identity", tensor_core=False, dims=None, B=None, precision="auto", backend=None,
        **agent_kw):
    dims = dims or ([64, 64, 32] if tensor_core else [4, 16, 3])
    B = B or (256 if tensor_core else 8)
    rng = np.random.RandomState(3)
    obs = torch.from_numpy(rng.standard_normal((B, dims[0])).astype(np.float32))
    tgt = torch.from_numpy(rng.dirichlet(np.ones(dims[-1]), B).astype(np.float32))
    be = backend or OracleBackend(tensor_core=tensor_core)
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
              policy_kwargs={"dims": dims, "hidden": hidden, "output": output},
              agent_kwargs=dict(obs=obs, target=tgt, loss="accuracy", **agent_kw), optimizer_kwargs={"lr": 0.01},
              noise_table_size=1 << 16, eval_precision=precision, _backend=be)
    es.log = lambda: None
    return es, be, obs, tgt


@pytest.mark.parametrize("hidden", ["relu", "tanh", "elu", "silu", "leaky_relu"])
def test_identity_output_is_fused_and_tanh_output_is_hooks(hidden):
    es = _es(hidden)[0]
    assert es._fused and es._act_code() == mlp.LOSS_ACCURACY | \
        {"relu": 0, "tanh": 1, "elu": 3, "silu": 4, "leaky_relu": 5}[hidden]
    assert not _es(hidden, "tanh")[0]._fused


def test_the_conv_vbn_policy_runs_in_hooks_mode():
    from test_xent_cpu import AtariPolicy
    g = torch.Generator().manual_seed(5)
    xref = torch.rand(2, 4, 84, 84, generator=g)
    es = E.ES(AtariPolicy, E.DeviceAgent, torch.optim.Adam, population_size=4, sigma=0.02,
              policy_kwargs=dict(n_actions=4, xref=xref), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 20,
              agent_kwargs=dict(obs=torch.rand(2, 4, 84, 84, generator=g),
                                target=F.one_hot(torch.tensor([0, 3]), 4).float(), loss="accuracy"),
              _backend=OracleBackend())
    assert es._is_conv and not es._fused


@pytest.mark.parametrize("tensor_core,dims,B,precision,want", [
    (False, None, None, "auto", "fp32"),
    (True, None, None, "auto", "f16"),
    (True, [784, 64, 10], 100, "auto", "fp32"),
    (True, [784, 64, 10], 100, "f16", "f16_any"),
    (True, None, None, "bf16", "bf16"),
    (True, None, None, "bf16s", "bf16s"),
    (True, None, None, "fp32", "fp32"),
])
def test_precision_follows_the_cross_entropy_and_the_code_reaches_the_backend(tensor_core, dims, B, precision, want):
    es, be, obs, tgt = _es("silu", tensor_core=tensor_core, dims=dims, B=B, precision=precision)
    assert es._precision == want
    es.train(n_steps=2)
    assert be.acts == {mlp.LOSS_ACCURACY | 4}
    with torch.no_grad():
        exact = float((es.policy(obs).argmax(1) == tgt.argmax(1)).float().mean())
    # the post-update rollout in the selected precision: within one or two rows of the fp32 torch forward
    assert abs(es.episode_reward - exact) <= 2.0 / obs.shape[0] + 1e-7


def test_a_cnn_classifier_is_fused_with_the_accuracy_code():
    x, y = image_task(24, (1, 12, 12), seed=2)
    dims = pack((1, 12, 12), [(4, 3, 2, 1), (6, 3, 2, 0)], [8, 4])
    be = OracleBackend()
    seen = []
    orig = be.eval_cnn

    def eval_cnn(*a, act=0, **k):
        seen.append(act)
        if (act & 0xff0000) == mlp.LOSS_ACCURACY:       # the stand-in's forward with the accuracy return
            return _cnn_accuracy(orig, *a, act=act, **k)
        return orig(*a, act=act, **k)
    be.eval_cnn = eval_cnn
    es = E.ES(cnn_policy_class(2, "relu"), E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05,
              policy_kwargs={"dims": dims}, agent_kwargs=dict(obs=x, target=y, loss="accuracy"),
              optimizer_kwargs={"lr": 0.02}, noise_table_size=1 << 14, _backend=be)
    es.log = lambda: None
    assert es._fused and es._is_cnn and es._act_code() == 2 << 24 | mlp.LOSS_ACCURACY
    es.train(n_steps=2)
    assert set(seen) == {2 << 24 | mlp.LOSS_ACCURACY}
    with torch.no_grad():
        assert es.episode_reward == float((es.policy(x).argmax(1) == y.argmax(1)).float().mean())


def _cnn_accuracy(orig, dims, theta, table, offsets, order, pairs, sigma, obs, target, ret_plus, ret_minus,
                  bc_plus=None, bc_minus=None, bc_obs=0, bc_dim=0, precision="fp32", act=0):
    from oracle import es_oracle as orc
    from _cnn_oracle import forward
    from _oracle_backend import _np
    rows = _np(theta)[None, :] if offsets is None else \
        orc.sample_population(_np(theta), _np(table), _np(offsets), sigma)[0]
    rets = np.array([mlp.accuracy_return(forward(r, dims, act & ~0xff0000, _np(obs)), _np(target)) for r in rows])
    if offsets is None:
        ret_plus[0] = float(rets[0])
        return
    ret_plus.copy_(torch.from_numpy(rets[:pairs]))
    ret_minus.copy_(torch.from_numpy(rets[pairs:]))


# ------------------------------------------------------------------ against the reference goldens
class HostAccuracyAgent:
    """A plain reference-protocol agent with the same rollout: forces hooks mode."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        self.inner = E.DeviceAgent(obs, target, bc_obs, bc_dim, loss="accuracy")

    def rollout(self, policy):
        return self.inner.rollout(policy)


@pytest.mark.parametrize("name", ["es_accuracy_p64.npz", "nsr_accuracy_p32.npz"])
def test_the_stand_in_reproduces_every_golden_return(name):
    """Every generation's returns (and, for NSR-ES, behaviour characteristics) from the recorded theta and offsets:
    accuracy counts on fp32 logits, bit for bit."""
    from oracle import es_oracle as orc
    g = load_golden(name)
    dims = [int(d) for d in g["dims"]]
    bc_obs, bc_dim = int(g["bc_obs"]), int(g["bc_dim"])
    for gen in range(len(g["returns"])):
        pop, _ = orc.sample_population(g["theta_before"][gen], g["table"], g["offsets"][gen], np.float32(g["sigma"]))
        rets, bcs = mlp.evaluate_population(pop, dims, g["obs"], g["target"], mlp.LOSS_ACCURACY, bc_obs=bc_obs,
                                            bc_dim=bc_dim)
        np.testing.assert_array_equal(rets, g["returns"][gen][:, 0])
        if bc_dim:
            np.testing.assert_allclose(bcs, _bcs_of(g, gen, pop, dims), rtol=1e-5, atol=1e-6)
    assert len(np.unique(g["returns"][0][:, 0])) < len(g["returns"][0])     # the returns tie


def _bcs_of(g, gen, pop, dims):
    """The reference's own logits through torch, as the golden's agent computed them."""
    out = []
    pol = MLP(dims, "relu")
    for row in pop:
        torch.nn.utils.vector_to_parameters(torch.from_numpy(row.copy()), pol.parameters())
        with torch.no_grad():
            out.append(pol(torch.from_numpy(g["obs"]))[:int(g["bc_obs"])].flatten()[:int(g["bc_dim"])].numpy())
    return np.stack(out)


@pytest.mark.parametrize("mode", ["fused", "hooks"])
def test_es_accuracy_first_generation_matches_the_reference_golden(mode):
    """Generation 0 scores the reference's initial theta: its returns equal the golden's in both modes.  Later
    generations depend on how ties among the returns are ranked (the engine's rule is stable by index)."""
    g = load_golden("es_accuracy_p64.npz")
    dims = [int(d) for d in g["dims"]]
    agent = E.DeviceAgent if mode == "fused" else HostAccuracyAgent
    akw = dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]))
    if mode == "fused":
        akw["loss"] = "accuracy"
    es = E.ES(MLP, agent, torch.optim.Adam, population_size=64, sigma=0.1,
              policy_kwargs={"dims": dims, "hidden": "relu"},
              agent_kwargs=akw, optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]),
              noise_seed=int(g["noise_seed"]), _backend=OracleBackend())
    rec = []
    es.log = lambda: rec.append(es.population_returns.copy())
    assert es._fused == (mode == "fused")
    es._table.copy_(torch.from_numpy(g["table"]))
    torch.nn.utils.vector_to_parameters(torch.from_numpy(g["theta0"].copy()), es.policy.parameters())
    if mode == "fused":
        es._slots[0].ensure_flat()
    es.train(n_steps=1)
    np.testing.assert_array_equal(rec[0][:, 0], g["returns"][0][:, 0])


# ------------------------------------------------------------------ fused against hooks, resume, minibatches
def _pair(dims=(5, 12, 4), B=40, seed=4, **agent_kw):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(B, dims[0], generator=g)
    tgt = F.one_hot(torch.randint(0, dims[-1], (B,), generator=g), dims[-1]).float()
    return obs, tgt


def _train(agent_cls, obs, tgt, n, seed=1, backend=None, **akw):
    torch.manual_seed(seed)
    es = E.ES(MLP, agent_cls, torch.optim.Adam, population_size=16, sigma=0.1,
              policy_kwargs={"dims": [obs.shape[1], 12, tgt.shape[1]], "hidden": "relu"},
              agent_kwargs=dict(obs=obs, target=tgt, **akw), optimizer_kwargs={"lr": 0.05},
              noise_table_size=1 << 14, noise_seed=7, _backend=backend or OracleBackend())
    rec = []
    es.log = lambda: rec.append((es.population_returns.copy(), float(es.episode_reward)))
    es.train(n_steps=n)
    return es, rec


def test_fused_equals_hooks_mode():
    obs, tgt = _pair()
    fused, a = _train(E.DeviceAgent, obs, tgt, 3, loss="accuracy")
    hooks, b = _train(HostAccuracyAgent, obs, tgt, 3)
    assert fused._fused and not hooks._fused
    for (ra, ea), (rb, eb) in zip(a, b):
        np.testing.assert_array_equal(ra[:, 0], rb[:, 0])
        assert ea == eb
    # the same ranks: the updates differ only by the fused Adam step's rounding against torch.optim.Adam's
    np.testing.assert_allclose(torch.nn.utils.parameters_to_vector(fused.policy.parameters()).detach().numpy(),
                               torch.nn.utils.parameters_to_vector(hooks.policy.parameters()).detach().numpy(),
                               rtol=1e-5, atol=1e-6)


def test_checkpoint_resume_is_bit_identical():
    obs, tgt = _pair(seed=6)
    a, a_rec = _train(E.DeviceAgent, obs, tgt, 4, loss="accuracy")
    b, _ = _train(E.DeviceAgent, obs, tgt, 2, loss="accuracy")
    sd = b.state_dict()
    torch.manual_seed(77)
    c = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=16, sigma=0.1,
             policy_kwargs={"dims": [5, 12, 4], "hidden": "relu"},
             agent_kwargs=dict(obs=obs, target=tgt, loss="accuracy"), optimizer_kwargs={"lr": 0.05},
             noise_table_size=1 << 14, noise_seed=7, _backend=OracleBackend())
    c.load_state_dict(sd)
    c_rec = []
    c.log = lambda: c_rec.append((c.population_returns.copy(), float(c.episode_reward)))
    c.train(n_steps=2)
    for sa, sc in zip(a._slots, c._slots):
        assert torch.equal(sa.theta, sc.theta) and torch.equal(sa.m, sc.m) and torch.equal(sa.v, sc.v)
    for (ra, ea), (rc, ec) in zip(a_rec[2:], c_rec):
        np.testing.assert_array_equal(ra, rc)
        assert ea == ec
    assert a.best_reward == c.best_reward


def test_minibatches_with_the_accuracy():
    """batch_size with loss="accuracy": fused, the accuracy code reaches the sampled evaluate, and generation g's
    returns score batch g (the same as hooks mode, which rolls out batch g on the host)."""
    obs, tgt = _pair(B=45, seed=8)
    be = OracleBackend()
    fused, a = _train(E.DeviceAgent, obs, tgt, 3, backend=be, loss="accuracy", batch_size=10, batch_seed=3)
    assert fused._fused and fused._sampling and be.acts == {mlp.LOSS_ACCURACY}

    torch.manual_seed(1)
    hooks = E.ES(MLP, E.DeviceAgent, torch.optim.SGD, population_size=16, sigma=0.1,     # SGD: hooks mode
                 policy_kwargs={"dims": [5, 12, 4], "hidden": "relu"},
                 agent_kwargs=dict(obs=obs, target=tgt, loss="accuracy", batch_size=10, batch_seed=3),
                 optimizer_kwargs={"lr": 0.05}, noise_table_size=1 << 14, noise_seed=7,
                 _backend=OracleBackend())
    assert not hooks._fused
    # generation 0's returns: the same initial theta and noise, the same batch 0
    rec = []
    hooks.log = lambda: rec.append(hooks.population_returns.copy())
    hooks.train(n_steps=1)
    np.testing.assert_array_equal(rec[0][:, 0], a[0][0][:, 0])
    i0 = torch.from_numpy(batch_indices(3, 0, 45, 10))
    assert all(r * 10 == round(r * 10) for r in a[0][0][:, 0])           # multiples of 1/B of the batch
    assert i0.shape == (10,)
