"""The streamed fp32 evaluate (eval_mlp_wide_kernel, estk_eval_mlp.cu) on the H100: the shapes the
shared-memory fp32 kernel cannot hold -- layers wider than 1080 and batches of more than 64 chunks --
against the oracle's fp32 forwards (tests/_act_oracle.py, tests/_xent_oracle.py), run-to-run and
order-independent bits, kernel selection read from torch.profiler, workspace growth and CUDA-graph
capture, and ES / NSR-ES runs through the public API."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import es_oracle as orc
import _act_oracle as act
import _xent_oracle as xo
from _xent_oracle import MLP, XentOracleBackend
from test_eval_mlp_act_gpu import _tc_problem, dev
import estorch_b200 as E

pytestmark = pytest.mark.gpu

WIDE, SMEM = "eval_mlp_wide_kernel", "eval_mlp_kernel"


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def _problem(dims, B, pairs, code, seed=3):
    n, table, theta, obs, tgt, offs = _tc_problem(dims, B, pairs, seed=seed)
    if code & xo.LOSS_XENT:
        tgt = np.eye(dims[-1], dtype=np.float32)[np.random.RandomState(seed).randint(0, dims[-1], B)]
    return n, table, theta, obs, tgt, offs


def _run(be, dims, theta, table, offs, sigma, obs, tgt, code, bc_obs=0, bc_dim=0, order=True):
    pairs = len(offs)
    ret = be.zeros(2 * pairs)
    bcp, bcm = (be.zeros(pairs, bc_dim), be.zeros(pairs, bc_dim)) if bc_dim else (None, None)
    o = dev(be, np.argsort(offs, kind="stable").astype(np.int32)) if order else None
    be.eval_mlp(dims, theta, table, dev(be, offs), o, pairs, sigma, obs, tgt, ret[:pairs], ret[pairs:], bcp, bcm,
                bc_obs, bc_dim, act=code)
    torch.cuda.synchronize()
    return ret.cpu().numpy(), (None if not bc_dim else np.concatenate([bcp.cpu().numpy(), bcm.cpu().numpy()]))


def _oracle(dims, theta, table, offs, sigma, obs, tgt, code, bc_obs=0, bc_dim=0):
    """Returns (and BCs) of pairs `offs`, [plus..., minus...], one pair at a time (wide rows are large)."""
    hidden, output = ("tanh" if code & act.ACT_TANH else "relu"), ("tanh" if code & act.ACT_OUT_TANH else "identity")
    rp, rm, bp, bm = [], [], [], []
    for off in offs:
        pop, _ = orc.sample_population(theta, table, np.array([off]), sigma)
        if code & xo.LOSS_XENT:
            r, b = xo.evaluate_population(pop, dims, obs, tgt, bc_obs, bc_dim, hidden)
        else:
            r, b = act.evaluate_population(pop, dims, obs, tgt, bc_obs, bc_dim, hidden, output)
        rp.append(r[0]); rm.append(r[1])
        if bc_dim:
            bp.append(b[0]); bm.append(b[1])
    return np.array(rp + rm), (np.stack(bp + bm) if bc_dim else None)


def _kernels(fn):
    """(names of the CUDA kernels the profiler saw while `fn` ran, fn's result).  CPU and CUDA activities, as
    in test_abi_gpu.py's launch count; a torch kernel launched first tells an empty trace from a missing launch."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").mul_(2.0)
        out = fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert any("eval_mlp" not in n for n in names), f"the profiler recorded no torch kernel of this window: {names}"
    return {n for n in names if "eval_mlp" in n}, out


# ------------------------------------------------------------------ returns against the oracle
# (dims, B, pairs, code, bc_obs, bc_dim): pairs x chunks of 64 observations > the SMs' persistent CTAs
SHAPES = [([1088, 64, 8], 256, 40, 0, 0, 0),
          ([16, 64, 2000], 256, 40, 0, 64, 256),
          ([32, 2048, 2048, 4], 128, 80, act.ACT_TANH | act.ACT_OUT_TANH, 0, 0),
          ([3072, 256, 10], 256, 40, xo.LOSS_XENT, 0, 0),
          ([32, 4096, 4096, 4], 128, 80, 0, 0, 0),
          ([784, 128, 10], 1024, 12, 0, 0, 0),
          ([784, 128, 10], 1000, 12, xo.LOSS_XENT, 8, 64),   # ragged last chunk
          ([784, 128, 10], 100, 4, 0, 0, 0),                  # the shared-memory kernel (13 chunks)
          ([784, 128, 10], 1, 4, 0, 0, 0),
          ([1088, 64, 8], 100, 150, act.ACT_TANH, 0, 0),      # ragged, one chunk per pair
          ([1088, 64, 8], 1, 150, xo.LOSS_XENT | act.ACT_TANH, 0, 0),
          ([784, 128, 10], 60000, 2, 0, 0, 0)]                # full-batch MNIST: 938 chunks per pair


@pytest.mark.parametrize("dims,B,pairs,code,bc_obs,bc_dim", SHAPES)
def test_wide_returns_vs_oracle(be, dims, B, pairs, code, bc_obs, bc_dim):
    n, table, theta, obs, tgt, offs = _problem(dims, B, pairs, code)
    th, tb, ob, tg = dev(be, theta), dev(be, table), dev(be, obs), dev(be, tgt)
    got, got_bc = _run(be, dims, th, tb, offs, 0.02, ob, tg, code, bc_obs, bc_dim)
    sel = np.unique(np.linspace(0, pairs - 1, min(pairs, 4)).astype(int))
    want, want_bc = _oracle(dims, theta, table, offs[sel], 0.02, obs, tgt, code, bc_obs, bc_dim)
    idx = np.concatenate([sel, pairs + sel])
    print(f"{dims} B={B} act={code:#x}: vs oracle {rel_err(got[idx], want):.2e}")
    assert rel_err(got[idx], want) < 1e-5
    if bc_dim:
        assert rel_err(got_bc[idx], want_bc) < 1e-5
    one = be.zeros(1)
    be.eval_mlp_center(dims, th, ob, tg, one, act=code)
    hidden, output = ("tanh" if code & act.ACT_TANH else "relu"), ("tanh" if code & act.ACT_OUT_TANH else "identity")
    y = act.mlp_forward(theta, dims, obs, hidden, output)
    w = float(xo.xent_return(y, tgt) if code & xo.LOSS_XENT else orc.synthetic_return(y, tgt))
    assert abs(float(one) - w) < 1e-5 * abs(w)


# ------------------------------------------------------------------ determinism
@pytest.mark.parametrize("dims,B,code", [([1088, 64, 8], 256, 0), ([3072, 256, 10], 200, xo.LOSS_XENT),
                                         ([784, 128, 10], 2000, act.ACT_TANH)])
def test_wide_bits_repeat_with_and_without_order_and_sigma0_is_centre(be, dims, B, code):
    pairs = 150
    n, table, theta, obs, tgt, offs = _problem(dims, B, pairs, code, seed=8)
    th, tb, ob, tg = dev(be, theta), dev(be, table), dev(be, obs), dev(be, tgt)
    a, _ = _run(be, dims, th, tb, offs, 0.02, ob, tg, code)
    b, _ = _run(be, dims, th, tb, offs, 0.02, ob, tg, code)
    c, _ = _run(be, dims, th, tb, offs, 0.02, ob, tg, code, order=False)
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(a, c)
    z, _ = _run(be, dims, th, tb, offs, 0.0, ob, tg, code)
    one = be.zeros(1)
    be.eval_mlp_center(dims, th, ob, tg, one, act=code)
    np.testing.assert_array_equal(z, np.full(2 * pairs, float(one), np.float32))


# ------------------------------------------------------------------ selection
@pytest.mark.parametrize("dims,B,kernel", [([1080, 64, 8], 256, SMEM), ([1088, 64, 8], 256, WIDE),
                                           ([784, 64, 10], 512, SMEM), ([784, 64, 10], 520, WIDE)])
def test_kernel_selection_by_name(dims, B, kernel):
    # In a fresh process: there the profile is the process's first.  After a profiling session has torn
    # CUPTI down, a later session in the same process may record no GPU activity at all (seen on the H100
    # as an empty trace, torch's own kernels included).
    code = """if True:
        import json, sys
        sys.path[:0] = sys.argv[3:]
        import numpy as np, torch
        from estorch_b200.backend import CudaBackend
        from test_eval_mlp_act_gpu import dev
        from test_eval_mlp_wide_gpu import _kernels, _problem, _run
        be = CudaBackend(torch.device("cuda", 0))
        dims, B = json.loads(sys.argv[1]), int(sys.argv[2])
        n, table, theta, obs, tgt, offs = _problem(dims, B, 4, 0)
        args = (dims, dev(be, theta), dev(be, table), offs, 0.02, dev(be, obs), dev(be, tgt), 0)
        want, _ = _run(be, *args)                        # workspace growth and module load outside the profile
        names, (got, _) = _kernels(lambda: _run(be, *args))
        print(json.dumps({"names": sorted(names), "same_bits": bool(np.array_equal(got, want))}))
    """
    tests = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", code, json.dumps(dims), str(B), os.path.dirname(tests), tests],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["same_bits"]
    assert len(out["names"]) == 1 and f"::{kernel}<" in out["names"][0], out


# ------------------------------------------------------------------ workspace
def test_wide_workspace_grows_refuses_under_capture_and_replays():
    from estorch_b200.backend import CudaBackend
    fresh = CudaBackend(torch.device("cuda", 0))
    dims, B, pairs = [32, 4096, 4096, 4], 128, 8
    n, table, theta, obs, tgt, offs = _problem(dims, B, pairs, 0, seed=5)
    th, tb, ob, tg, of = dev(fresh, theta), dev(fresh, table), dev(fresh, obs), dev(fresh, tgt), dev(fresh, offs)
    ret = fresh.zeros(2 * pairs)

    def call():
        fresh.eval_mlp(dims, th, tb, of, None, pairs, 0.02, ob, tg, ret[:pairs], ret[pairs:])
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match=r"estk_status -4\).*captured"):
        with torch.cuda.graph(graph):
            call()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    call()                                               # eagerly it grows: 2 x 4096 x 128 floats per CTA
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 >= 2 * 4096 * 128 * 4 * min(pairs * 2, fresh.sm_count)   # pairs x 2 chunks
    eager = ret.cpu().numpy().copy()
    ret.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    ret.zero_()
    graph.replay()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(ret.cpu().numpy(), eager)
    want, _ = _oracle(dims, theta, table, offs[:1], 0.02, obs, tgt, 0)
    assert rel_err(eager[[0, pairs]], want) < 1e-5


# ------------------------------------------------------------------ public API
def _xent_es(backend, mode_graph, monkeypatch):
    monkeypatch.setenv("ESTORCH_B200_GRAPH", mode_graph)
    rng = np.random.RandomState(2)
    dims, B = [3072, 256, 10], 256
    obs = torch.from_numpy(rng.standard_normal((B, dims[0])).astype(np.float32))
    tgt = torch.from_numpy(np.eye(10, dtype=np.float32)[rng.randint(0, 10, B)])
    rec = []

    class R(E.ES):
        def log(self):
            rec.append((self.population_returns.copy(), self.episode_reward,
                        self._slots[0].theta.detach().cpu().numpy().copy()))
    torch.manual_seed(6)
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.02, policy_kwargs={"dims": dims},
           agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy"), optimizer_kwargs={"lr": 0.01},
           noise_table_size=1 << 21, _backend=backend)
    return es, rec


def test_es_wide_xent_fused_fp32_vs_oracle_standin_and_graph(monkeypatch):
    es, rec = _xent_es(None, "0", monkeypatch)
    assert es._fused and es._be.name == "cuda" and es._precision == "fp32"
    table = es._table.cpu()
    es.train(n_steps=3)
    ref, rref = _xent_es(XentOracleBackend(), "0", monkeypatch)
    ref._table.copy_(table)
    ref.train(n_steps=3)
    (r_c, ep_c, _), (r_o, ep_o, _) = rec[0], rref[0]
    print(f"gen 0: returns vs stand-in {rel_err(r_c[:, 0], r_o[:, 0]):.2e}")
    assert rel_err(r_c[:, 0], r_o[:, 0]) < 1e-5
    assert abs(ep_c - ep_o) < 1e-5 * abs(ep_o)
    for gen in range(3):
        # ranks may swap between returns closer than the two evaluations' difference; Adam moves an entry
        # by at most lr per generation
        assert np.abs(rec[gen][2] - rref[gen][2]).max() <= 2 * 0.01 * (gen + 1) + 1e-6
        assert np.all(np.isfinite(rec[gen][0])) and np.isfinite(rec[gen][1])
    g, rg = _xent_es(None, "1", monkeypatch)
    g.train(n_steps=6)
    e, re_ = _xent_es(None, "0", monkeypatch)
    e.train(n_steps=6)
    assert sum(isinstance(v, tuple) for v in g.__dict__.get("_graphs", {}).values()) >= 1
    for a, b in zip(rg, re_):
        np.testing.assert_array_equal(a[0], b[0])
        np.testing.assert_array_equal(a[2], b[2])
        assert a[1] == b[1]


def test_nsr_es_wide_hidden_trains_fused():
    rng = np.random.RandomState(5)
    dims, B = [24, 2048, 4], 256
    obs = torch.from_numpy(rng.standard_normal((B, dims[0])).astype(np.float32))
    tgt = torch.from_numpy(rng.uniform(-1, 1, (B, dims[-1])).astype(np.float32))
    rec = []

    class R(E.NSR_ES):
        def log(self):
            rec.append((self.population_returns.copy(), self.episode_reward))
    np.random.seed(1)
    torch.manual_seed(1)
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.02, policy_kwargs={"dims": dims},
           agent_kwargs=dict(obs=obs, target=tgt, bc_obs=64, bc_dim=256), optimizer_kwargs={"lr": 0.01},
           noise_table_size=1 << 20)
    assert es._fused and es._be.name == "cuda" and es._precision == "fp32"
    es.train(n_steps=3)
    assert len(rec) == 3
    for r, ep in rec:
        assert np.all(np.isfinite(r)) and np.isfinite(ep)
