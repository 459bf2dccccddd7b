"""Minibatches drawn on the H100 (estk_sample_batch, estk_batch.cu): the kernel's rows equal the host restatement
``batch_indices`` over a sweep of (N, B, seed, g), the gathered rows are the dataset's bytes for every row size and
alignment, a captured call replays the next batches as the counter advances, ``ES.train`` with ``batch_size`` is
bit-identical to the same rows fed through ``next_batch`` in every evaluate mode (and replays from a CUDA graph),
resume, two GPUs where present, and the minibatch example learns."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import estorch_b200 as E
from estorch_b200 import batch_indices
from conftest import ROOT
from _mlp_oracle import MLP

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def _bits(t):
    return t.contiguous().view(torch.int32)


def _random_bits(shape, seed, dev, offset=0):
    """A float32 tensor of ``shape`` holding random bit patterns (NaNs and denormals included), starting
    ``offset`` floats into its allocation (offset 1: 4-byte but not 8- or 16-byte aligned rows)."""
    n = int(np.prod(shape))
    g = torch.Generator().manual_seed(seed)
    raw = torch.randint(-2**31, 2**31 - 1, (n + offset,), generator=g, dtype=torch.int64).to(torch.int32)
    return raw.view(torch.float32).to(dev)[offset:].view(shape)


def _state(be, generation):
    from estorch_b200.backend import new_state, write_state
    s = new_state(be.device)
    write_state(s, generation=generation)
    return s


# ------------------------------------------------------------------ the rows
SWEEP = [(1, 1), (7, 3), (97, 10), (97, 97), (256, 256), (4096, 100), (60000, 256), (65537, 4096),
         ((1 << 26) + 3, 1000)]
GENS = [0, 1, 2, 5, 59, (1 << 32) // 256 + 1, (1 << 40) - 3, (1 << 40) + 7]


@pytest.mark.parametrize("n,b", SWEEP)
def test_kernel_indices_equal_the_restatement(be, n, b):
    obs = torch.zeros(n, 1, device=be.device)
    dst, tdst = be.zeros(b, 1), be.zeros(b, 1)
    idx = be.zeros(b, dtype=torch.int64)
    for seed in (0, 12345, (1 << 64) - 1):
        for g in GENS + [(n // b) or 1, (n + b - 1) // b]:        # an epoch boundary inside or at a batch edge
            be.sample_batch(seed, None, g, obs, dst, obs, tdst, idx)
            want = batch_indices(seed, g, n, b)
            assert np.array_equal(idx.cpu().numpy(), want), (seed, g)
            s = _state(be, g - 1)                                  # the same g read from estk_state + 1
            be.sample_batch(seed, s, 1, obs, dst, obs, tdst, idx)
            assert np.array_equal(idx.cpu().numpy(), want), (seed, g, "state")


@pytest.mark.parametrize("row,trow,offset", [(1, 1, 0), (3, 2, 0), (3, 5, 1), (784, 10, 0), (784, 10, 1),
                                             (3072, 10, 0), (3 * 32 * 32, 7, 2), (1025, 1, 0), (5000, 3, 1)])
def test_gathered_rows_are_the_dataset_bytes(be, row, trow, offset):
    n, b = 1000, 256
    obs, tgt = _random_bits((n, row), 1, be.device, offset), _random_bits((n, trow), 2, be.device, offset)
    dst, tdst = be.alloc(b, row), be.alloc(b, trow)
    idx = be.zeros(b, dtype=torch.int64)
    for g in (0, 3, 17):                                          # 17 * 256 straddles an epoch of 1000 rows
        be.sample_batch(9, None, g, obs, dst, tgt, tdst, idx)
        want = torch.from_numpy(batch_indices(9, g, n, b)).to(be.device)
        assert torch.equal(idx, want)
        assert torch.equal(_bits(dst), _bits(obs[want])) and torch.equal(_bits(tdst), _bits(tgt[want]))


def test_sequences_are_gathered_whole(be):
    n, b, T = 300, 64, 9
    obs, tgt = _random_bits((n, T, 5), 3, be.device), _random_bits((n, T, 2), 4, be.device)
    dst, tdst = be.alloc(b, T, 5), be.alloc(b, T, 2)
    be.sample_batch(1, None, 6, obs, dst, tgt, tdst)
    want = torch.from_numpy(batch_indices(1, 6, n, b)).to(be.device)
    assert torch.equal(_bits(dst), _bits(obs[want])) and torch.equal(_bits(tdst), _bits(tgt[want]))


def test_only_the_destination_rows_are_written(be):
    n, b = 500, 100
    obs, tgt = _random_bits((n, 3), 5, be.device), _random_bits((n, 1), 6, be.device)
    guard = torch.full((b * 3 + 8,), 7.0, device=be.device)
    dst = guard[4:4 + b * 3].view(b, 3)
    tdst = be.alloc(b, 1)
    be.sample_batch(2, None, 4, obs, dst, tgt, tdst)
    assert bool((guard[:4] == 7).all()) and bool((guard[4 + b * 3:] == 7).all())


def test_a_captured_call_replays_the_next_batches(be):
    n, b, g0, k = 700, 64, 40, 6
    obs, tgt = _random_bits((n, 12), 7, be.device), _random_bits((n, 3), 8, be.device)
    dst, tdst = be.alloc(b, 12), be.alloc(b, 3)
    state = _state(be, g0)
    launches = be.launches
    side = torch.cuda.Stream(be.device)
    side.wait_stream(torch.cuda.current_stream(be.device))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        graph.capture_begin()
        be.sample_batch(3, state, 0, obs, dst, tgt, tdst)
        graph.capture_end()
    torch.cuda.current_stream(be.device).wait_stream(side)
    assert be.launches == launches + 1
    gen = state.view(torch.int64)[:1]                              # estk_state.generation
    for i in range(k):
        graph.replay()
        want = torch.from_numpy(batch_indices(3, g0 + i, n, b)).to(be.device)
        assert torch.equal(_bits(dst), _bits(obs[want])) and torch.equal(_bits(tdst), _bits(tgt[want])), i
        gen += 1


def test_refusals_launch_nothing(be):
    obs, dst = be.zeros(10, 2), be.zeros(4, 2)
    launches = be.launches
    for kw in [dict(gen_host=-1), dict(dst=be.zeros(11, 2))]:
        with pytest.raises(RuntimeError, match=r"estk_status -1\)"):
            be.sample_batch(0, None, kw.get("gen_host", 0), obs, kw.get("dst", dst), obs, kw.get("dst", dst))
    torch.cuda.synchronize()
    assert be.launches == launches and bool((dst == 0).all())


# ------------------------------------------------------------------ ES.train
def _streamed(obs, tgt, seed, b, base):
    """A ``base`` agent class fed the same rows through the next_batch host hook: fresh pinned tensors, kept alive
    so that no two generations hand over the same host addresses (each generation then runs eagerly)."""
    class Streamed(base):
        def __init__(self, **kw):
            i0 = torch.from_numpy(batch_indices(seed, 0, obs.shape[0], b))
            super().__init__(obs[i0], tgt[i0], **kw)
            self.handed = []

        def next_batch(self, step):
            idx = torch.from_numpy(batch_indices(seed, step, obs.shape[0], b))
            self.handed.append((obs[idx].pin_memory(), tgt[idx].pin_memory()))
            return self.handed[-1]
    return Streamed


def _train(policy, agent, agent_kwargs, policy_kwargs, n_steps=5, **kw):
    # free the earlier cases' engines now (``es.log`` closes over its engine, a cycle): a collection during a
    # later graph capture would release their pinned batches there and invalidate the capture
    gc.collect()
    torch.manual_seed(11)
    es = E.ES(policy, agent, torch.optim.Adam, population_size=kw.pop("P", 64), sigma=0.02,
              policy_kwargs=policy_kwargs, agent_kwargs=agent_kwargs, optimizer_kwargs={"lr": 0.01},
              noise_table_size=1 << 22, noise_seed=3, **kw)
    rec = []
    es.log = lambda: rec.append((es.population_returns.copy(), es.episode_reward))
    es.train(n_steps=n_steps)
    torch.cuda.synchronize()
    return es, rec


def _cases():
    from _cnn_oracle import image_task, pack, policy_class as cnn_policy
    from _rnn_oracle import policy_class as rnn_policy
    from test_api_gpu import AtariPolicy
    g = torch.Generator().manual_seed(21)
    reg = lambda n, i, o: (torch.randn(n, i, generator=g), 0.5 * torch.randn(n, o, generator=g))
    onehot = lambda n, i, c: (torch.randn(n, i, generator=g),
                              torch.nn.functional.one_hot(torch.randint(0, c, (n,), generator=g), c).float())
    img = image_task(90, (1, 12, 12), seed=4)
    seq = (torch.randn(60, 6, 3, generator=g), torch.rand(60, 6, 2, generator=g))
    xref = torch.rand(4, 4, 84, 84, generator=g)
    frames = (torch.rand(12, 4, 84, 84, generator=g), torch.randn(12, 4, generator=g))
    return {   # name: (policy, agent, (obs, target), B, policy_kwargs, engine kwargs, expected precision)
        "mlp_auto_f16": (MLP, E.DeviceAgent, reg(1000, 64, 32), 256, {"dims": [64, 128, 32]}, {}, "f16"),
        "mlp_fp32": (MLP, E.DeviceAgent, reg(300, 5, 3), 50, {"dims": [5, 32, 3]}, {"eval_precision": "fp32"}, "fp32"),
        "mlp_f16_any_xent": (MLP, E.DeviceAgent, onehot(400, 40, 10), 100, {"dims": [40, 48, 10]},
                             {"eval_precision": "f16", "loss": "cross_entropy"}, "f16_any"),
        "cnn": (cnn_policy(2, "relu"), E.DeviceAgent, img, 20,
                {"dims": pack((1, 12, 12), [(4, 3, 2, 1), (6, 3, 2, 0)], [8, 4])}, {"loss": "cross_entropy"}, "fp32"),
        "gru": (rnn_policy("gru", True), E.SequenceAgent, seq, 16, {"dims": (3, 16, 2)}, {}, "fp32"),
        "lstm": (rnn_policy("lstm", False), E.SequenceAgent, seq, 16, {"dims": (3, 16, 2)}, {}, "fp32"),
        "conv_vbn_fp32": (AtariPolicy, E.DeviceAgent, frames, 4, {"n_actions": 4, "xref": xref}, {}, "fp32"),
        "conv_vbn_f16": (AtariPolicy, E.DeviceAgent, frames, 4, {"n_actions": 4, "xref": xref},
                         {"eval_precision": "f16"}, "f16"),
    }


@pytest.mark.parametrize("name", ["mlp_auto_f16", "mlp_fp32", "mlp_f16_any_xent", "cnn", "gru", "lstm",
                                  "conv_vbn_fp32", "conv_vbn_f16"])
def test_sampled_training_equals_the_same_rows_through_next_batch(name):
    policy, agent, (obs, tgt), b, pkw, kw, precision = _cases()[name]
    kw = dict(kw)
    akw = {"loss": kw.pop("loss")} if "loss" in kw else {}
    a, a_rec = _train(policy, agent, dict(obs=obs, target=tgt, batch_size=b, batch_seed=8, **akw), pkw, **kw)
    assert a._fused and a._sampling and a._precision == precision
    assert any(isinstance(v, tuple) for v in a.__dict__.get("_graphs", {}).values()), "no CUDA-graph replay"
    c, c_rec = _train(policy, _streamed(obs, tgt, 8, b, agent), akw, pkw, **kw)
    assert c._fused and not c._sampling and c._precision == precision
    assert torch.equal(a._slots[0].theta, c._slots[0].theta)
    assert len(a_rec) == len(c_rec) == 5
    for (ra, ea), (rc, ec) in zip(a_rec, c_rec):
        np.testing.assert_array_equal(ra, rc)
        assert ea == ec
    assert a.best_reward == c.best_reward


def test_checkpoint_resume_is_bit_identical_on_the_device():
    policy, agent, (obs, tgt), b, pkw, kw, _ = _cases()["mlp_auto_f16"]
    akw = dict(obs=obs, target=tgt, batch_size=b, batch_seed=2)
    a, a_rec = _train(policy, agent, akw, pkw, n_steps=4)
    b_, _ = _train(policy, agent, akw, pkw, n_steps=2)
    sd = b_.state_dict()
    torch.manual_seed(99)
    c = E.ES(policy, agent, torch.optim.Adam, population_size=64, sigma=0.02, policy_kwargs=pkw, agent_kwargs=akw,
             optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 22, noise_seed=3)
    c.load_state_dict(sd)
    rec = []
    c.log = lambda: rec.append((c.population_returns.copy(), c.episode_reward))
    c.train(n_steps=2)
    for x, y in zip((a._slots[0].theta, a._slots[0].m, a._slots[0].v), (c._slots[0].theta, c._slots[0].m,
                                                                        c._slots[0].v)):
        assert torch.equal(x, y)
    for (ra, ea), (rc, ec) in zip(a_rec[2:], rec):
        np.testing.assert_array_equal(ra, rc)
        assert ea == ec


_TWO_GPU = """if True:
    import os, sys, numpy as np, torch
    sys.path[:0] = sys.argv[2:]
    import estorch_b200 as E
    from test_minibatch_gpu import MLP
    g = torch.Generator().manual_seed(5)
    x, y = torch.randn(5000, 64, generator=g), torch.randn(5000, 32, generator=g)
    torch.manual_seed(1)
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=256, sigma=0.02,
              policy_kwargs={"dims": [64, 128, 32]}, agent_kwargs=dict(obs=x, target=y, batch_size=256),
              optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 22)
    es.log = lambda: None
    es.train(n_steps=6)
    np.savez(os.path.join(sys.argv[1], f"rank{es.rank}.npz"), theta=es._slots[0].theta.cpu().numpy(),
             returns=es.population_returns, world=es.n_workers)
    es.close()
"""


def test_two_gpu_replicas_stay_bit_identical(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = [subprocess.Popen([sys.executable, "-c", _TWO_GPU, str(tmp_path), ROOT, os.path.join(ROOT, "tests")],
                              env=dict(os.environ, RANK=str(r), WORLD_SIZE="2", LOCAL_RANK=str(r),
                                       MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port)),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT) for r in range(2)]
    outs = [p.communicate(timeout=900)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o[-3000:]
    r0, r1 = (np.load(os.path.join(tmp_path, f"rank{r}.npz")) for r in range(2))
    assert int(r0["world"]) == 2
    np.testing.assert_array_equal(r0["theta"], r1["theta"])
    np.testing.assert_array_equal(r0["returns"], r1["returns"])


def test_the_minibatch_example_learns():
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import minibatch_classifier as ex
    acc0, acc1 = ex.main(**ex.TEST_SETTINGS)
    print(f"full-dataset accuracy {acc0:.3f} -> {acc1:.3f}")
    assert acc1 >= ex.TEST_ACCURACY and acc1 > acc0 + 0.3
