"""Recurrent policies on sequence batches without a GPU: SequenceAgent's validation and rollout, mode selection,
the reference goldens reproduced through ES / NSR-ES on the oracle stand-in (tests/_seq_oracle.py), fused mode
against hooks mode, evaluate launches per generation, checkpoint / resume, a gloo world-2 run, and the sequence
codes in the header and the library's support probe."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import estorch_b200.estorch as E
from estorch_b200 import DeviceAgent, SequenceAgent, _capi
from conftest import ROOT, load_golden, rel_err
from _rnn_oracle import CELL_GRU, CELL_LSTM, policy_class
from _oracle_backend import OracleBackend
from _seq_oracle import memoryless_best, recall_dataset, seq_outputs32, seq_returns32
from test_population_rnn_cpu import _load_theta, _Rec, check_es_golden, check_nsr_golden

DIMS = (3, 8, 2)


def _data(B=5, T=4, seed=9):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T, DIMS[0], generator=g), torch.rand(B, T, DIMS[2], generator=g) - 0.5


def _es(cls=E.ES, cell="gru", out_tanh=True, optimizer=torch.optim.Adam, agent=SequenceAgent, agent_kwargs=None,
        P=16, dims=DIMS, **kw):
    obs, tgt = _data()
    es = cls(policy_class(cell, out_tanh), agent, optimizer, population_size=P, sigma=0.05,
             policy_kwargs={"dims": dims}, agent_kwargs=agent_kwargs or dict(obs=obs, target=tgt),
             optimizer_kwargs={"lr": 0.02}, noise_table_size=1 << 13, _backend=OracleBackend(), **kw)
    es.log = lambda: None
    return es


# ------------------------------------------------------------------ the agent
def test_agent_validation():
    obs, tgt = _data()
    for bad in ((obs[:, 0], tgt), (obs, tgt[:, 0]), (obs, tgt[:4]), (obs, tgt[:, :3]), (obs[:, :0], tgt[:, :0])):
        with pytest.raises(ValueError, match="obs must be"):
            SequenceAgent(*bad)
    with pytest.raises(ValueError, match="loss"):
        SequenceAgent(obs, tgt, loss="hinge")
    with pytest.raises(ValueError, match="cross_entropy"):
        SequenceAgent(obs, tgt, loss="cross_entropy")               # negative class weights
    with pytest.raises(ValueError, match="bc_obs"):
        SequenceAgent(obs, tgt, bc_obs=2)
    ag = SequenceAgent(obs.double(), tgt.double())
    assert ag.obs.shape == (5, 4, 3) and ag.target.shape == (5, 4, 2) and ag.obs.dtype == torch.float32
    assert ag.next_batch(0) is None and isinstance(ag, DeviceAgent)


@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_rollout_runs_the_policy_over_every_step_with_its_state(cell):
    obs, tgt = _data()
    torch.manual_seed(0)
    pol = policy_class(cell, True)(DIMS)
    ys, state = [], None
    with torch.no_grad():
        for t in range(obs.shape[1]):
            y, state = pol(obs[:, t], state)
            ys.append(y)
    y = torch.stack(ys, 1)
    assert SequenceAgent(obs, tgt).rollout(pol) == float(-((y - tgt) ** 2).mean())
    r, bc = SequenceAgent(obs, tgt, bc_obs=2, bc_dim=11).rollout(pol)
    np.testing.assert_array_equal(bc, y[:2].flatten()[:11].numpy())
    # cross-entropy: the mean over the B*T steps; all-zero target rows add 0
    ro, rt = recall_dataset()
    pol = policy_class(cell, False)((4, 8, 3))
    with torch.no_grad():
        ys, state = [], None
        for t in range(ro.shape[1]):
            y, state = pol(ro[:, t], state)
            ys.append(y)
    last = torch.log_softmax(ys[-1], 1)
    want = float((rt[:, -1] * last).sum(1).sum() / (ro.shape[0] * ro.shape[1]))
    assert abs(SequenceAgent(ro, rt, loss="cross_entropy").rollout(pol) - want) < 1e-7


def test_rollout_of_a_memoryless_policy():
    obs, tgt = _data()
    lin = torch.nn.Linear(3, 2)
    with torch.no_grad():
        want = float(-((lin(obs) - tgt) ** 2).mean())
    assert abs(SequenceAgent(obs, tgt).rollout(lin) - want) < 1e-7


# ------------------------------------------------------------------ mode selection
@pytest.mark.parametrize("cell", ["gru", "lstm"])
@pytest.mark.parametrize("loss", ["mse", "cross_entropy"])
def test_fused_mode_is_selected_for_a_recurrent_policy_on_sequences(cell, loss):
    obs, tgt = _data()
    if loss == "cross_entropy":
        tgt = tgt.abs()
    es = _es(cell=cell, out_tanh=loss == "mse", agent_kwargs=dict(obs=obs, target=tgt, loss=loss))
    assert es._fused and es._is_rnn and not es._population and es._precision == "fp32"
    assert es._act_code() == (CELL_GRU if cell == "gru" else CELL_LSTM) | \
        (0x100 if loss == "mse" else _capi.ESTK_LOSS_XENT)


class _Hooks(E.ES):
    def _after_optimize(self, policy):          # any overridden hook selects hooks mode
        super()._after_optimize(policy)


@pytest.mark.parametrize("case", ["xent_tanh", "mlp_policy", "device_agent", "sgd", "hook", "shape", "k"])
def test_hooks_mode_serves_everything_else(case):
    obs, tgt = _data()
    if case == "xent_tanh":
        es = _es(agent_kwargs=dict(obs=obs, target=tgt.abs(), loss="cross_entropy"))
    elif case == "mlp_policy":
        from test_api_cpu import MLP
        es = E.ES(MLP, SequenceAgent, torch.optim.Adam, population_size=8, sigma=0.05, policy_kwargs={"dims": [3, 8, 2]},
                  agent_kwargs=dict(obs=obs, target=tgt), noise_table_size=1 << 13, _backend=OracleBackend())
    elif case == "device_agent":
        es = _es(agent=DeviceAgent, agent_kwargs=dict(obs=obs[:, 0], target=tgt[:, 0]))
    elif case == "sgd":
        es = _es(optimizer=torch.optim.SGD)
    elif case == "hook":
        es = _es(cls=_Hooks)
    elif case == "shape":
        es = _es(dims=(4, 8, 2))
    else:
        es = _es(cls=E.NS_ES, k=33, agent_kwargs=dict(obs=obs, target=tgt, bc_obs=1, bc_dim=8))
    assert not es._fused and not es._population


def test_fused_mode_refuses_a_tensor_core_precision():
    for prec in ("f16", "bf16", "bf16s"):
        with pytest.raises(ValueError, match="fp32 only"):
            _es(eval_precision=prec)
    assert _es(eval_precision="fp32")._fused


# ------------------------------------------------------------------ the oracle's reduction
def test_restatement_of_the_reduction():
    """seq_returns32 is the documented order, and agrees with the float64 return of the same outputs."""
    rng = np.random.RandomState(0)
    y = rng.standard_normal((3, 4, 5, 2)).astype(np.float32)
    tg = rng.standard_normal((4, 5, 2)).astype(np.float32)
    got = seq_returns32(y, tg, False)
    f = np.float32
    for m in range(3):
        S = f(0)
        for b in range(4):
            L = f(0)
            for t in range(5):
                s = f(0)
                for c in range(2):
                    d = f(y[m, b, t, c] - tg[b, t, c])
                    s = f(np.float64(d) * d + s)
                L = f(L + s)
            S = f(S + L)
        assert got[m] == f(-(S / f(40)))
    w = -((y.astype(np.float64) - tg[None]) ** 2).mean((1, 2, 3))
    assert np.abs(got - w).max() < 1e-6
    onehot = np.eye(2, dtype=np.float32)[rng.randint(0, 2, (4, 5))]
    onehot[:, :-1] = 0                                     # only the last step scored
    x = seq_returns32(y, onehot, True)
    lsm = y[:, :, -1] - np.log(np.exp(y[:, :, -1].astype(np.float64)).sum(-1, keepdims=True))
    assert np.abs(x - (onehot[None, :, -1] * lsm).sum(-1).sum(1) / 20).max() < 1e-6


# ------------------------------------------------------------------ the reference goldens
def run_es_seq_golden(backend):
    """ES with the GRU policy in fused mode from es_seq_gru_p16.npz's start; returns (instance, fixture)."""
    g = load_golden("es_seq_gru_p16.npz")

    class R(_Rec, E.ES):
        pass
    es = R(policy_class("gru", True), SequenceAgent, torch.optim.Adam, population_size=16, sigma=float(g["sigma"]),
           policy_kwargs={"dims": tuple(int(d) for d in g["dims"])}, optimizer_kwargs={"lr": 0.01},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"])),
           noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]), _backend=backend)
    es.rec = []
    assert es._fused and es._is_rnn and not es._population
    es._table.copy_(torch.from_numpy(g["table"]).to(es._dev))
    _load_theta(es.policy, g["theta0"])
    es._slots[0].ensure_flat()
    es.train(n_steps=3)
    return es, g


def run_nsr_seq_golden(backend):
    """NSR-ES with the LSTM policy, cross-entropy on the recall dataset, from nsr_seq_lstm_p8.npz's start."""
    g = load_golden("nsr_seq_lstm_p8.npz")

    class R(_Rec, E.NSR_ES):
        pass
    np.random.seed(123)
    es = R(policy_class("lstm", False), SequenceAgent, torch.optim.Adam, population_size=8, sigma=float(g["sigma"]),
           policy_kwargs={"dims": tuple(int(d) for d in g["dims"])}, optimizer_kwargs={"lr": 0.01},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]),
                             bc_obs=int(g["bc_obs"]), bc_dim=int(g["bc_dim"]), loss="cross_entropy"),
           noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]), _backend=backend)
    es.rec = []
    assert es._fused and es._is_rnn
    es._table.copy_(torch.from_numpy(g["table"]).to(es._dev))
    for i, (p, _) in enumerate(es.meta_population):
        _load_theta(p, g["meta_theta0"][i])
        es._slots[i].ensure_flat()
        es._slots[i].push_theta()
    es._archive = [a.copy() for a in g["archive0"]]
    np.random.seed(123)
    es.train(n_steps=len(g["grad"]))
    return es, g


def test_es_gru_sequence_matches_reference_golden():
    check_es_golden(*run_es_seq_golden(OracleBackend()))


def test_nsr_lstm_cross_entropy_sequence_matches_reference_golden():
    check_nsr_golden(*run_nsr_seq_golden(OracleBackend()))


def test_the_recall_dataset_needs_memory():
    obs, tgt = recall_dataset()
    assert obs.shape == (3, 6, 4) and tgt.shape == (3, 6, 3) and float(tgt[:, :-1].abs().sum()) == 0.0
    uniform = np.zeros((1, 3, 6, 3), np.float32)          # the best a memoryless policy can do: equal logits
    assert abs(float(seq_returns32(uniform, tgt.numpy(), True)[0]) - memoryless_best()) < 1e-7
    perfect = np.where(tgt.numpy()[None] > 0, np.float32(30), np.float32(0))
    assert float(seq_returns32(perfect, tgt.numpy(), True)[0]) > -1e-6


# ------------------------------------------------------------------ fused against hooks mode
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_fused_mode_matches_hooks_mode(cell):
    runs = []
    for cls in (E.ES, _Hooks):
        torch.manual_seed(5)
        es = _es(cls=cls, cell=cell, P=8)
        rec = []
        es.log = lambda es=es, rec=rec: rec.append((es.population_returns.copy(), es.episode_reward))
        es.train(n_steps=3)
        theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().numpy()
        runs.append((es._fused, rec, theta))
    (fused, f_rec, f_theta), (hooks, h_rec, h_theta) = runs
    assert fused and not hooks
    for (rf, ef), (rh, eh) in zip(f_rec, h_rec):
        assert rel_err(rf[:, 0], rh[:, 0]) < 1e-5
        assert abs(ef - eh) < 1e-5 * abs(eh)
    assert rel_err(f_theta, h_theta) < 2e-4


def test_the_stand_in_evaluate_is_the_restatement_of_the_outputs():
    es = _es(P=8)
    slot = es._slots[0]
    es._draw_offsets()
    ret = torch.zeros(8)
    es._be.eval_rnn_seq(DIMS, slot.theta, es._table, es._offsets, es._order, 4, es.sigma, es._obs, es._tgt,
                        ret[:4], ret[4:], act=es._act_code())
    from oracle import es_oracle as orc
    rows, _ = orc.sample_population(slot.theta.numpy(), es._table.numpy(), es._offsets.numpy(), es.sigma)
    y = seq_outputs32(rows, "gru", DIMS, es._obs.numpy(), True)
    np.testing.assert_array_equal(ret.numpy(), seq_returns32(y, es._tgt.numpy(), False))


# ------------------------------------------------------------------ launches, resume
def test_one_population_and_one_centre_evaluate_per_generation():
    es = _es()
    es.train(n_steps=3)
    assert es._be.seq_calls == 2 * 3 and es._be.act_calls == 0
    ns = _es(cls=E.NSR_ES, agent_kwargs=dict(obs=_data()[0], target=_data()[1], bc_obs=2, bc_dim=8))
    calls0 = ns._be.seq_calls                     # the meta-population's initial archive entries
    ns.train(n_steps=2)
    # per generation: the population, the meta-population's centres (_select_slot), the updated centre
    assert ns._be.seq_calls - calls0 == 2 * (1 + ns.meta_population_size + 1)


@pytest.mark.parametrize("cls,cell,bc", [(E.ES, "gru", False), (E.NSR_ES, "lstm", True)])
def test_checkpoint_resume_is_bit_identical(cls, cell, bc):
    obs, tgt = _data()
    kw = dict(obs=obs, target=tgt, bc_obs=2, bc_dim=8) if bc else None

    def make(seed):
        torch.manual_seed(seed)
        return _es(cls=cls, cell=cell, agent_kwargs=kw)
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


# ------------------------------------------------------------------ two processes over gloo
def test_world2_equals_world1(tmp_path):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="1")
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "_seq_dist_worker.py"),
                                       str(tmp_path)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
    outs = [p.communicate(timeout=600)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o[-3000:]
    r0, r1 = (np.load(os.path.join(tmp_path, f"rank{r}.npz")) for r in range(2))
    assert int(r0["world"]) == 2 and int(r0["pairs_local"]) == 4
    for k in ("theta", "returns", "episode"):
        np.testing.assert_array_equal(r0[k], r1[k])
    from _seq_dist_worker import run
    es, _ = run()
    assert es.n_workers == 1
    assert rel_err(r0["returns"][:, 0], es.population_returns[:, 0]) < 1e-5
    assert rel_err(r0["theta"], es._slots[0].theta.numpy()) < 1e-5


# ------------------------------------------------------------------ ABI
SEQ_CODES = [c | rest for c in (CELL_GRU, CELL_LSTM) for rest in (0, 1 << 8, _capi.ESTK_LOSS_XENT)]


def test_header_documents_the_sequence_codes():
    header = open(os.path.join(ROOT, "include", "estk.h")).read()
    for text in ("Recurrent sequence evaluate", "dims[3] = T >= 1", "obs is [B][T][in] and target [B][T][out]",
                 "29 in all", "the sequence codes add 6", "35 in all", "-(S / (float)(B*T*out))",
                 "-(S / (float)(B*T))", "sum of L_b over b in ascending order", "T chained ESTK_ACTIONS launches"):
        assert text in header, text


def test_support_probe_returns_0_for_the_sequence_codes():
    from estorch_b200.backend import mlp_desc
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = _capi.load()
    for code in SEQ_CODES:
        for prec in (_capi.ESTK_PREC_FP32, _capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S,
                     _capi.ESTK_PREC_F16_ANY):
            for dims, T in (([64, 64, 32], 8), ([64, 64, 32], 0), ([64, 128, 64, 32], 0)):
                d = mlp_desc(dims, code, steps=T)
                assert lib.estk_eval_mlp_supported(C.byref(d), prec, 256) == 0, (hex(code), prec, dims, T)
