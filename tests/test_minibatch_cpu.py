"""Minibatches drawn on the device, without a GPU: the host restatement ``batch_indices`` (the oracle of the
kernel's rows), ``DeviceAgent`` / ``SequenceAgent`` with ``batch_size``, mode selection, the fused generation on
the stand-in backend against the same rows fed through ``next_batch``, hooks mode, resume, a gloo world of 2, and
the refusals of ``estk_sample_batch``."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import estorch_b200.estorch as E
from estorch_b200 import DeviceAgent, SequenceAgent, _capi, batch_indices
from conftest import ROOT, rel_err
from _batch_oracle import dataset
from _cnn_oracle import image_task, pack, policy_class as cnn_policy_class
from _oracle_backend import OracleBackend
from _rnn_oracle import policy_class as rnn_policy_class
from _mlp_oracle import MLP


# ------------------------------------------------------------------ the restatement
CASES = [(1, 1), (5, 5), (97, 10), (97, 97), (64, 16), (64, 7), (65, 16), (257, 64), (1 << 12, 100)]


@pytest.mark.parametrize("n,b", CASES)
def test_every_epoch_is_a_permutation_of_the_rows(n, b):
    stream = np.concatenate([batch_indices(7, g, n, b) for g in range((3 * n + b - 1) // b)])
    for e in range(3):
        assert np.array_equal(np.sort(stream[e * n:(e + 1) * n]), np.arange(n)), e


@pytest.mark.parametrize("n,b", CASES)
def test_rows_are_distinct_within_a_batch_that_stays_in_one_epoch(n, b):
    for g in range(40):
        idx = batch_indices(3, g, n, b)
        assert idx.dtype == np.int64 and idx.shape == (b,) and idx.min() >= 0 and idx.max() < n
        if (g * b) // n == (g * b + b - 1) // n:
            assert len(set(idx.tolist())) == b, g


@pytest.mark.parametrize("n,b", [(97, 10), (1 << 16, 256), ((1 << 16) + 1, 256), (60000, 256), ((1 << 31) - 1, 64)])
@pytest.mark.parametrize("g", [0, 1, (1 << 32) // 256 + 3, (1 << 40) - 1, (1 << 40) + 12345])
def test_a_batch_is_its_slice_of_the_epoch_permutations(n, b, g):
    """Batch g is positions g*B .. g*B + B - 1 of pi_0, pi_1, ...; batch_indices(seed, e, N, N) is pi_e itself
    (the positions of epoch e), also where g*B passes 2^32 and the batch straddles two epochs."""
    e0, r0 = divmod(g * b, n)
    if n > 1 << 20:            # a whole epoch of 2^31 rows is too large to list: check range and distinctness
        idx = batch_indices(11, g, n, b)
        assert idx.min() >= 0 and idx.max() < n and (r0 + b > n or len(set(idx.tolist())) == b)
        return
    perm = np.concatenate([batch_indices(11, e0, n, n), batch_indices(11, e0 + 1, n, n)])
    assert np.array_equal(batch_indices(11, g, n, b), perm[r0:r0 + b])


def test_deterministic_in_seed_and_generation_and_seeds_differ():
    a = batch_indices(5, 9, 1000, 64)
    assert np.array_equal(a, batch_indices(5, 9, 1000, 64))
    assert not np.array_equal(a, batch_indices(6, 9, 1000, 64))
    assert not np.array_equal(a, batch_indices(5, 10, 1000, 64))
    assert not np.array_equal(batch_indices(0, 0, 1000, 1000), np.arange(1000))
    assert np.array_equal(batch_indices(-1, 3, 50, 7), batch_indices((1 << 64) - 1, 3, 50, 7))


def test_the_restatement_refuses_what_the_kernel_refuses():
    for args in [(0, 0, 0, 1), (0, 0, 1 << 31, 1), (0, 0, 10, 0), (0, 0, 10, 11), (0, -1, 10, 2)]:
        with pytest.raises(ValueError):
            batch_indices(*args)


# ------------------------------------------------------------------ agents
def test_device_agent_with_batch_size_holds_the_dataset_and_batch_g():
    x, y = dataset(50, 3, 2)
    ag = DeviceAgent(x, y, batch_size=8, batch_seed=4)
    assert ag.batch_size == 8 and ag.batch_seed == 4
    assert torch.equal(ag.dataset_obs, x) and torch.equal(ag.dataset_target, y)
    i0 = torch.from_numpy(batch_indices(4, 0, 50, 8))
    assert torch.equal(ag.obs, x[i0]) and torch.equal(ag.target, y[i0])
    ag.set_generation(13)
    i13 = torch.from_numpy(batch_indices(4, 13, 50, 8))
    assert torch.equal(ag.obs, x[i13]) and torch.equal(ag.target, y[i13])
    policy = MLP([3, 4, 2])
    with torch.no_grad():
        want = float(-((policy(x[i13]) - y[i13]) ** 2).mean())
    assert ag.rollout(policy) == want


def test_sequence_agent_with_batch_size_samples_whole_sequences():
    g = torch.Generator().manual_seed(2)
    x, y = torch.randn(30, 5, 3, generator=g), torch.rand(30, 5, 2, generator=g)
    ag = SequenceAgent(x, y, batch_size=6, batch_seed=1)
    assert ag.dataset_obs.shape == (30, 5, 3) and ag.dataset_target.shape == (30, 5, 2)
    ag.set_generation(7)
    idx = torch.from_numpy(batch_indices(1, 7, 30, 6))
    assert torch.equal(ag.obs, x[idx]) and torch.equal(ag.target, y[idx])


def test_an_agent_without_batch_size_is_unchanged():
    x, y = dataset(20, 3, 2)
    ag = DeviceAgent(x, y, 2, 4, loss="mse")
    assert set(vars(ag)) == {"obs", "target", "loss", "bc_obs", "bc_dim"}
    assert torch.equal(ag.obs, x) and torch.equal(ag.target, y) and (ag.bc_obs, ag.bc_dim) == (2, 4)
    assert ag.batch_size is None and ag.dataset_obs is None
    with pytest.raises(ValueError, match="batch_size"):
        ag.set_generation(1)
    sq = SequenceAgent(x.reshape(20, 1, 3), y.reshape(20, 1, 2))
    assert set(vars(sq)) == {"obs", "target", "loss", "bc_obs", "bc_dim"} and sq.obs.shape == (20, 1, 3)


@pytest.mark.parametrize("bad", [0, -1, 21, 2.0, "4", True, None])
def test_batch_size_must_be_an_int_between_1_and_n(bad):
    x, y = dataset(20, 3, 2)
    if bad is None:
        assert DeviceAgent(x, y, batch_size=np.int64(20)).batch_size == 20
        return
    with pytest.raises(ValueError, match="batch_size"):
        DeviceAgent(x, y, batch_size=bad)
    with pytest.raises(ValueError, match="batch_size"):
        SequenceAgent(x.reshape(20, 1, 3), y.reshape(20, 1, 2), batch_size=bad)


def test_a_dataset_of_2_31_rows_is_refused_before_it_is_copied():
    big = torch.zeros(1, 1).expand(1 << 31, 1)           # no storage behind the rows
    with pytest.raises(ValueError, match="too large"):
        DeviceAgent(big, big, batch_size=4)
    with pytest.raises(ValueError, match="too large"):
        SequenceAgent(big.unsqueeze(1), big.unsqueeze(1), batch_size=4)


def test_batch_size_with_a_behaviour_characteristic_is_refused():
    x, y = dataset(20, 3, 2)
    for bc in [(2, 4), (2, 0), (0, 4)]:
        with pytest.raises(ValueError, match="behaviour characteristic"):
            DeviceAgent(x, y, *bc, batch_size=4)
    with pytest.raises(ValueError, match="behaviour characteristic"):
        SequenceAgent(x.reshape(20, 1, 3), y.reshape(20, 1, 2), 1, 2, batch_size=4)


def test_the_existing_rules_apply_to_the_whole_dataset():
    x, y = dataset(20, 3, 4, classes=True)
    y_bad = y.clone()
    y_bad[17, 0] = -1.0                                   # outside most batches: still refused
    with pytest.raises(ValueError, match="cross_entropy"):
        DeviceAgent(x, y_bad, loss="cross_entropy", batch_size=4)
    with pytest.raises(ValueError, match="obs must be"):
        DeviceAgent(x, y[:19], batch_size=4)
    with pytest.raises(ValueError, match="loss"):
        DeviceAgent(x, y, loss="hinge", batch_size=4)
    assert DeviceAgent(x, y, loss="cross_entropy", batch_size=4).loss == "cross_entropy"


# ------------------------------------------------------------------ mode selection
def _es(cls=E.ES, policy=MLP, dims=(3, 8, 2), n=40, b=8, backend=None, agent=DeviceAgent, agent_kwargs=None,
        optimizer=torch.optim.Adam, **kw):
    if agent_kwargs is None:
        x, y = dataset(n, dims[0], dims[-1])
        agent_kwargs = dict(obs=x, target=y, batch_size=b, batch_seed=3)
    return cls(policy, agent, optimizer, population_size=kw.pop("P", 8), sigma=0.05,
               policy_kwargs=kw.pop("policy_kwargs", {"dims": list(dims)}), agent_kwargs=agent_kwargs,
               optimizer_kwargs={"lr": 0.02}, noise_table_size=1 << 13, noise_seed=5,
               _backend=backend or OracleBackend(), **kw)


def test_es_adam_with_a_sampling_agent_is_fused_for_an_mlp_a_cnn_and_a_sequence_agent():
    es = _es()
    assert es._fused and es._sampling and es._data_obs.shape == (40, 3) and es._obs.shape == (8, 3)
    x, y = image_task(30, (1, 12, 12), seed=2)
    cnn = _es(policy=cnn_policy_class(2, "relu"), backend=OracleBackend(),
              policy_kwargs={"dims": pack((1, 12, 12), [(4, 3, 2, 1), (6, 3, 2, 0)], [8, 4])},
              agent_kwargs=dict(obs=x, target=y, loss="cross_entropy", batch_size=6))
    assert cnn._fused and cnn._is_cnn and cnn._sampling and cnn._obs.shape == (6, 1, 12, 12)
    g = torch.Generator().manual_seed(9)
    seq = _es(policy=rnn_policy_class("gru", True), backend=OracleBackend(), agent=SequenceAgent,
              policy_kwargs={"dims": (3, 8, 2)},
              agent_kwargs=dict(obs=torch.randn(25, 4, 3, generator=g), target=torch.rand(25, 4, 2, generator=g),
                                batch_size=5))
    assert seq._fused and seq._is_rnn and seq._sampling and seq._obs.shape == (5, 4, 3)
    hooks = _es(optimizer=torch.optim.SGD)
    assert not hooks._fused and hooks._sampling and hooks._data_obs is None


def test_the_post_update_rollout_is_never_deferred_while_sampling():
    """On the tensor-core evaluate a fixed batch folds the post-update rollout into the next launch; a minibatch
    does not, because the next launch scores another batch."""
    runs = {}
    for b in (None, 256):
        x, y = dataset(512, 64, 32)
        kw = dict(obs=x[:256], target=y[:256]) if b is None else dict(obs=x, target=y, batch_size=b)
        es = _es(dims=(64, 64, 32), agent_kwargs=kw, backend=OracleBackend(tensor_core=True),
                 eval_precision="bf16", log_interval=4)
        es.n_steps, es.step = 8, 0
        runs[b] = es._defers_centre()
    assert runs == {None: True, 256: False}


def test_an_agent_cannot_have_both_batch_size_and_next_batch():
    class Streaming(DeviceAgent):
        def next_batch(self, step):
            return None
    x, y = dataset(40, 3, 2)
    with pytest.raises(ValueError, match="next_batch"):
        _es(agent=Streaming, agent_kwargs=dict(obs=x, target=y, batch_size=8))
    assert not _es(agent=Streaming, agent_kwargs=dict(obs=x[:8], target=y[:8]))._sampling


def test_the_ns_family_stays_on_fixed_batches():
    x, y = dataset(40, 3, 2)
    with pytest.raises(ValueError, match="behaviour characteristic"):
        _es(cls=E.NSR_ES, agent_kwargs=dict(obs=x, target=y, bc_obs=2, bc_dim=4, batch_size=8))


# ------------------------------------------------------------------ the fused generation
def _streamed(dataset_obs, dataset_target, seed, b):
    """A DeviceAgent class fed the same rows by the next_batch host hook."""
    class Streamed(DeviceAgent):
        def __init__(self, **kw):
            i0 = torch.from_numpy(batch_indices(seed, 0, dataset_obs.shape[0], b))
            super().__init__(dataset_obs[i0], dataset_target[i0], **kw)

        def next_batch(self, step):
            idx = torch.from_numpy(batch_indices(seed, step, dataset_obs.shape[0], b))
            return dataset_obs[idx], dataset_target[idx]
    return Streamed


def _run(es, n):
    rec = []
    es.log = lambda: rec.append((es.population_returns.copy(), float(es.episode_reward)))
    es.train(n_steps=n)
    return rec, es._slots[0].theta.clone()


def test_fused_sampling_equals_the_same_rows_through_next_batch():
    x, y = dataset(37, 3, 2, seed=4)
    torch.manual_seed(1)
    be = OracleBackend()
    a_rec, a_theta = _run(_es(agent_kwargs=dict(obs=x, target=y, batch_size=8, batch_seed=3), backend=be), 3)
    assert be.batch_calls == 3
    torch.manual_seed(1)
    b = _es(agent=_streamed(x, y, 3, 8), agent_kwargs={}, backend=OracleBackend())
    assert b._fused and not b._sampling
    b_rec, b_theta = _run(b, 3)
    assert torch.equal(a_theta, b_theta)
    for (ra, ea), (rb, eb) in zip(a_rec, b_rec):
        np.testing.assert_array_equal(ra, rb)
        assert ea == eb
    # and not the fixed batch 0
    torch.manual_seed(1)
    i0 = torch.from_numpy(batch_indices(3, 0, 37, 8))
    c_rec, c_theta = _run(_es(agent_kwargs=dict(obs=x[i0], target=y[i0]), backend=OracleBackend()), 3)
    np.testing.assert_array_equal(c_rec[0][0], a_rec[0][0])
    assert not torch.equal(c_theta, a_theta)


def test_hooks_mode_rolls_out_generation_g_on_batch_g():
    x, y = dataset(30, 3, 2, seed=6)
    seen = []

    class Recording(DeviceAgent):
        def rollout(self, policy):
            seen.append(self.obs.clone())
            return super().rollout(policy)
    es = _es(agent=Recording, agent_kwargs=dict(obs=x, target=y, batch_size=7, batch_seed=2),
             optimizer=torch.optim.SGD)
    assert not es._fused
    es.log = lambda: None
    es.train(n_steps=3)
    per = es.population_size + 1                           # P member rollouts, then the post-update one
    assert len(seen) == 3 * per
    for g in range(3):
        want = x[torch.from_numpy(batch_indices(2, g, 30, 7))]
        assert all(torch.equal(o, want) for o in seen[g * per:(g + 1) * per]), g


def test_checkpoint_resume_is_bit_identical():
    x, y = dataset(29, 3, 2, seed=8)
    kw = dict(obs=x, target=y, batch_size=6, batch_seed=9)

    def make(seed):
        torch.manual_seed(seed)
        return _es(agent_kwargs=kw)
    a = make(1)
    a_rec, _ = _run(a, 4)
    b = make(1)
    _run(b, 2)
    sd = b.state_dict()
    c = make(77)
    c.load_state_dict(sd)
    c_rec, _ = _run(c, 2)
    for sa, sc in zip(a._slots, c._slots):
        assert torch.equal(sa.theta, sc.theta) and torch.equal(sa.m, sc.m) and torch.equal(sa.v, sc.v)
    for (ra, ea), (rc, ec) in zip(a_rec[2:], c_rec):
        np.testing.assert_array_equal(ra, rc)
        assert ea == ec
    assert a.best_reward == c.best_reward


def test_world2_equals_world1(tmp_path):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), OMP_NUM_THREADS="1")
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "_batch_dist_worker.py"),
                                       str(tmp_path)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
    outs = [p.communicate(timeout=600)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o[-3000:]
    r0, r1 = (np.load(os.path.join(tmp_path, f"rank{r}.npz")) for r in range(2))
    assert int(r0["world"]) == 2 and int(r0["batch_calls"]) == 3
    for k in ("theta", "returns", "episode"):
        np.testing.assert_array_equal(r0[k], r1[k])
    from _batch_dist_worker import run
    es, _ = run()
    assert es.n_workers == 1
    # the two ranks sum the gradient in another order: the same run up to fp32 rounding
    assert rel_err(r0["returns"][:, 0], es.population_returns[:, 0]) < 1e-5
    assert rel_err(r0["theta"], es._slots[0].theta.numpy()) < 1e-5


# ------------------------------------------------------------------ the C ABI
def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


def test_the_sampler_is_declared_apart_from_the_core_header_and_bound_to_it():
    """estk_sample_batch lives in include/estk_batch.h (which includes estk.h); the binding's table of it agrees
    with that header, and the core header and its table do not list it."""
    import re
    header = open(os.path.join(ROOT, "include", "estk_batch.h")).read()
    assert '#include "estk.h"' in header and "0x6261746368657321" in header
    declared = sorted(set(re.findall(r"ESTK_API\s+[\w\s\*]+?\b(estk_\w+)\s*\(", header)))
    assert declared == sorted(_capi.BATCH_SIGNATURES) == ["estk_sample_batch"]
    m = re.search(r"\bestk_sample_batch\s*\(([^)]*)\)", header)
    assert len(m.group(1).split(",")) == len(_capi.BATCH_SIGNATURES["estk_sample_batch"]) == 14
    assert "estk_sample_batch" not in open(os.path.join(ROOT, "include", "estk.h")).read()
    assert "estk_sample_batch" not in _capi.SIGNATURES
    lib = _lib()
    assert hasattr(lib, "estk_sample_batch") and lib.estk_sample_batch.argtypes is not None


FAKE = C.c_void_p(256)          # never dereferenced: every call below is refused before the context is read


def _sample(**over):
    """estk_sample_batch on a well-formed call (N = 10, B = 4, 3-float rows) with the arguments in ``over``
    replaced; the destinations and index_out are host arrays that a refused call must leave untouched."""
    bufs = {k: np.full(shape, 7, dt) for k, shape, dt in
            [("obs_dst", (4, 3), np.float32), ("tgt_dst", (4, 2), np.float32), ("index_out", 4, np.int64)]}
    ptr = {k: C.c_void_p(v.ctypes.data) for k, v in bufs.items()}
    a = dict(ctx=FAKE, seed=1, state=None, gen_host=0, n=10, b=4, obs_src=FAKE, obs_row=3, obs_dst=ptr["obs_dst"],
             tgt_src=FAKE, tgt_row=2, tgt_dst=ptr["tgt_dst"], index_out=ptr["index_out"])
    a.update(over)
    rc = _lib().estk_sample_batch(a["ctx"], a["seed"], a["state"], a["gen_host"], a["n"], a["b"], a["obs_src"],
                                  a["obs_row"], a["obs_dst"], a["tgt_src"], a["tgt_row"], a["tgt_dst"],
                                  a["index_out"], None)
    untouched = all((v == 7).all() for v in bufs.values())
    return rc, untouched


@pytest.mark.parametrize("over", [
    dict(ctx=None), dict(n=0), dict(n=-5), dict(n=1 << 31), dict(n=1 << 40), dict(b=0), dict(b=-1), dict(b=11),
    dict(n=3, b=4), dict(obs_row=0), dict(obs_row=-3), dict(tgt_row=0), dict(tgt_row=-1), dict(obs_src=None),
    dict(tgt_src=None), dict(obs_dst=None), dict(tgt_dst=None), dict(gen_host=-1), dict(gen_host=-(1 << 62))],
    ids=lambda d: ",".join(f"{k}={v}" for k, v in d.items()))
def test_refusals_return_invalid_and_write_nothing(over):
    rc, untouched = _sample(**over)
    assert rc == -1 and untouched
    assert b"estk_sample_batch" in _lib().estk_last_error()
