"""ESTK_PREC_F16_ANY on the H100: the F16 arithmetic for every MLP shape.  The streamed wgmma kernel
(estk_eval_mlp_tc_stream.cu) against the f16 emulation and the exact fp32 forward (tests/_act_oracle.py,
tests/_xent_oracle.py), bit agreement with the cluster kernel, run-to-run bits, the ABI, workspace growth
under CUDA graphs, kernel selection and the launch counter read from torch.profiler, and ES / NSR-ES runs
with eval_precision="f16" through the public API."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import es_oracle as orc
import _act_oracle as act
import _xent_oracle as xo
from _xent_oracle import MLP
from test_eval_mlp_act_gpu import _set_theta, _tc_problem, dev
import estorch_b200 as E

pytestmark = pytest.mark.gpu

STREAM, CLUSTER, SPLIT = "eval_mlp_tc_stream_kernel", "eval_mlp_tc_kernel", "split_obs_f16_kernel"
ALL_CODES = (0, act.ACT_TANH, act.ACT_OUT_TANH, act.ACT_TANH | act.ACT_OUT_TANH, xo.LOSS_XENT,
             xo.LOSS_XENT | act.ACT_TANH)


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def _problem(dims, B, pairs, code, seed=23):
    n, table, theta, obs, tgt, offs = _tc_problem(dims, B, pairs, seed=seed)
    if code & xo.LOSS_XENT:
        tgt = np.eye(dims[-1], dtype=np.float32)[np.random.RandomState(seed).randint(0, dims[-1], B)]
    return n, table, theta, obs, tgt, offs


class Dev:
    """A problem's buffers on the device, with the exact fp16 copy of the table."""
    def __init__(self, be, theta, table, obs, tgt):
        self.th, self.tb, self.ob, self.tg = dev(be, theta), dev(be, table), dev(be, obs), dev(be, tgt)
        self.tb16 = be.alloc(table.size, dtype=torch.float16)
        assert be.shadow_f16(self.tb, self.tb16) == 0


def _run(be, dims, d, offs, sigma, code, bc_obs=0, bc_dim=0, order=True, precision="f16_any", obs=None, tgt=None,
         centre_out=None):
    pairs = len(offs)
    ret = be.zeros(2 * pairs)
    bcp, bcm = (be.zeros(pairs, bc_dim), be.zeros(pairs, bc_dim)) if bc_dim else (None, None)
    o = dev(be, np.argsort(offs, kind="stable").astype(np.int32)) if order else None
    be.eval_mlp(dims, d.th, d.tb, dev(be, offs), o, pairs, sigma, d.ob if obs is None else obs,
                d.tg if tgt is None else tgt, ret[:pairs], ret[pairs:], bcp, bcm, bc_obs, bc_dim, precision=precision,
                table16=d.tb16, act=code, centre_out=centre_out)
    torch.cuda.synchronize()
    return ret.cpu().numpy(), (None if not bc_dim else np.concatenate([bcp.cpu().numpy(), bcm.cpu().numpy()]))


def _centre(be, dims, d, code, bc_obs=0, bc_dim=0):
    one, bc = be.zeros(1), (be.zeros(bc_dim) if bc_dim else None)
    be.eval_mlp_center(dims, d.th, d.ob, d.tg, one, bc, bc_obs, bc_dim, precision="f16_any", act=code)
    torch.cuda.synchronize()
    return float(one), (None if bc is None else bc.cpu().numpy())


def _oracle(dims, theta, table, offs, sigma, obs, tgt, code, bc_obs, bc_dim, precision):
    """Returns (and BCs) of pairs `offs`, [plus..., minus...], one pair at a time."""
    hidden, output = ("tanh" if code & act.ACT_TANH else "relu"), ("tanh" if code & act.ACT_OUT_TANH else "identity")
    rp, rm, bp, bm = [], [], [], []
    for off in offs:
        pop, _ = orc.sample_population(theta, table, np.array([off]), sigma)
        if code & xo.LOSS_XENT:
            r, b = xo.evaluate_population(pop, dims, obs, tgt, bc_obs, bc_dim, hidden, precision)
        else:
            r, b = act.evaluate_population(pop, dims, obs, tgt, bc_obs, bc_dim, hidden, output, precision)
        rp.append(r[0]); rm.append(r[1])
        if bc_dim:
            bp.append(b[0]); bm.append(b[1])
    return np.array(rp + rm), (np.stack(bp + bm) if bc_dim else None)


def _centre_oracle(dims, theta, obs, tgt, code, precision):
    hidden, output = ("tanh" if code & act.ACT_TANH else "relu"), ("tanh" if code & act.ACT_OUT_TANH else "identity")
    y = act.FORWARD[precision](theta, list(dims), obs, hidden, output)
    return float(xo.xent_return(y, tgt) if code & xo.LOSS_XENT else orc.synthetic_return(y, tgt))


# ------------------------------------------------------------------ returns against the emulation and fp32
# (dims, B, pairs, code, bc_obs, bc_dim); every one is a shape ESTK_PREC_F16 refuses
SHAPES = [([4, 64, 64, 2], 1, 8, 0, 0, 0),
          ([4, 64, 64, 2], 256, 8, 0, 0, 0),
          ([784, 256, 10], 100, 4, xo.LOSS_XENT, 0, 0),
          ([784, 256, 10], 1000, 4, xo.LOSS_XENT, 8, 64),        # ragged last chunk
          ([3072, 512, 10], 256, 3, xo.LOSS_XENT, 0, 0),
          ([320, 64, 32], 256, 4, 0, 0, 0),
          ([64, 1024, 1024, 32], 128, 3, 0, 0, 0),
          ([24, 64, 64, 4], 256, 6, 0, 64, 256),
          ([784, 128, 10], 60000, 1, 0, 0, 0)]                  # full-batch MNIST: 938 chunks per pair
SHAPES += [([33, 200, 70, 10], 100, 3, c, 16, 100) for c in ALL_CODES]


@pytest.mark.parametrize("dims,B,pairs,code,bc_obs,bc_dim", SHAPES)
def test_f16_any_returns_vs_emulation_and_fp32(be, dims, B, pairs, code, bc_obs, bc_dim):
    assert not be.eval_supports_f16(dims, B, act=code) and be.eval_supports_f16_any(dims, B, act=code)
    n, table, theta, obs, tgt, offs = _problem(dims, B, pairs, code)
    d = Dev(be, theta, table, obs, tgt)
    got, got_bc = _run(be, dims, d, offs, 0.02, code, bc_obs, bc_dim)
    sel = np.unique(np.linspace(0, pairs - 1, min(pairs, 2)).astype(int))
    idx = np.concatenate([sel, pairs + sel])
    emu, emu_bc = _oracle(dims, theta, table, offs[sel], 0.02, obs, tgt, code, bc_obs, bc_dim, "f16")
    exact, exact_bc = _oracle(dims, theta, table, offs[sel], 0.02, obs, tgt, code, bc_obs, bc_dim, "fp32")
    print(f"{dims} B={B} act={code:#x}: vs emulation {rel_err(got[idx], emu):.2e}, vs fp32 {rel_err(got[idx], exact):.2e}")
    assert np.all(np.isfinite(got))
    assert rel_err(got[idx], emu) < 1e-5
    # B = 1 with two outputs: the return is the mean of two squared errors, so the fp16 rounding of the
    # weights (2^-12 relative) does not average out over observations (measured 1.4e-4, DESIGN section 9)
    assert rel_err(got[idx], exact) < (3e-4 if B == 1 else 3e-5)
    if bc_dim:
        assert rel_err(got_bc[idx], emu_bc) < 2e-3 and rel_err(got_bc[idx], exact_bc) < 2e-3
    one, _ = _centre(be, dims, d, code)
    assert abs(one - _centre_oracle(dims, theta, obs, tgt, code, "f16")) < 1e-5 * abs(one)


# ------------------------------------------------------------------ agreement with the cluster kernel
@pytest.mark.parametrize("dims", [[64, 256, 64], [128, 512, 512, 288]])
def test_streamed_bcs_equal_cluster_kernel_bits(be, dims):
    """B = 255 runs the streamed kernel, B = 256 the cluster kernel: the same pre-activations, bit for bit."""
    n, table, theta, obs, tgt, offs = _problem(dims, 256, 3, 0)
    d = Dev(be, theta, table, obs, tgt)
    bc_dim = 255 * dims[-1]
    _, cl = _run(be, dims, d, offs, 0.02, 0, 255, bc_dim, precision="f16")
    _, st = _run(be, dims, d, offs, 0.02, 0, 255, bc_dim, obs=d.ob[:255], tgt=d.tg[:255])
    np.testing.assert_array_equal(st, cl)
    # on a rule shape "f16_any" is the cluster kernel: returns, BCs and the folded centre are F16's bits
    c16, cany = be.zeros(1), be.zeros(1)
    r16, b16 = _run(be, dims, d, offs, 0.02, 0, 64, 256, precision="f16", centre_out=c16)
    rany, bany = _run(be, dims, d, offs, 0.02, 0, 64, 256, centre_out=cany)
    np.testing.assert_array_equal(rany, r16)
    np.testing.assert_array_equal(bany, b16)
    assert float(c16) == float(cany)


# ------------------------------------------------------------------ determinism and special cases
@pytest.mark.parametrize("dims,B,code", [([784, 256, 10], 200, xo.LOSS_XENT), ([320, 64, 32], 100, act.ACT_TANH),
                                         ([24, 64, 64, 4], 300, act.ACT_OUT_TANH)])
def test_bits_repeat_with_and_without_order_and_sigma0_is_centre(be, dims, B, code):
    pairs = 150
    n, table, theta, obs, tgt, offs = _problem(dims, B, pairs, code, seed=8)
    d = Dev(be, theta, table, obs, tgt)
    a, abc = _run(be, dims, d, offs, 0.02, code, 8, 64)
    b, bbc = _run(be, dims, d, offs, 0.02, code, 8, 64)
    c, cbc = _run(be, dims, d, offs, 0.02, code, 8, 64, order=False)
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(a, c)
    np.testing.assert_array_equal(abc, bbc)
    np.testing.assert_array_equal(abc, cbc)
    z, zbc = _run(be, dims, d, offs, 0.0, code, 8, 64)
    one, bc1 = _centre(be, dims, d, code, 8, 64)
    np.testing.assert_array_equal(z, np.full(2 * pairs, one, np.float32))
    np.testing.assert_array_equal(zbc, np.broadcast_to(bc1, zbc.shape))


# ------------------------------------------------------------------ ABI
def test_abi_centre_fold_alignment_and_codes(be):
    dims, B = [320, 64, 32], 100
    n, table, theta, obs, tgt, offs = _problem(dims, B, 2, 0)
    d = Dev(be, theta, table, obs, tgt)
    ret, c_out = be.zeros(4).fill_(7.0), be.zeros(1).fill_(7.0)
    launches = be.launches
    with pytest.raises(RuntimeError, match=r"estk_status -3\).*centre_return_out"):
        be.eval_mlp(dims, d.th, d.tb, dev(be, offs), None, 2, 0.02, d.ob, d.tg, ret[:2], ret[2:], precision="f16_any",
                    table16=d.tb16, centre_out=c_out)
    torch.cuda.synchronize()
    assert be.launches == launches
    assert torch.equal(ret, torch.full_like(ret, 7.0)) and float(c_out) == 7.0
    unaligned = be.zeros(B * dims[0] + 1)[1:].view(B, dims[0])
    unaligned.copy_(d.ob)
    with pytest.raises(RuntimeError, match=r"estk_status -1\)"):
        be.eval_mlp(dims, d.th, d.tb, dev(be, offs), None, 2, 0.02, unaligned, d.tg, ret[:2], ret[2:],
                    precision="f16_any", table16=d.tb16)
    with pytest.raises(RuntimeError, match=r"estk_status -1\)"):      # a population needs table16
        be.eval_mlp(dims, d.th, d.tb, dev(be, offs), None, 2, 0.02, d.ob, d.tg, ret[:2], ret[2:], precision="f16_any")
    for bad in (2, 0x200, xo.LOSS_XENT | act.ACT_OUT_TANH, 1 << 24):
        assert not be.eval_supports_f16_any(dims, B, act=bad)
        with pytest.raises(RuntimeError, match=r"estk_status -3\)"):
            be.eval_mlp(dims, d.th, d.tb, dev(be, offs), None, 2, 0.02, d.ob, d.tg, ret[:2], ret[2:],
                        precision="f16_any", table16=d.tb16, act=bad)
    torch.cuda.synchronize()
    assert torch.equal(ret, torch.full_like(ret, 7.0))
    # ESTK_PREC_F16 keeps its rule
    assert not be.eval_supports_f16(dims, 256)
    with pytest.raises(RuntimeError, match=r"estk_status -3\).*not supported"):
        be.eval_mlp(dims, d.th, d.tb, dev(be, offs), None, 2, 0.02, d.ob, d.tg, ret[:2], ret[2:], precision="f16",
                    table16=d.tb16)


# ------------------------------------------------------------------ workspace
def test_workspace_grows_refuses_under_capture_and_earlier_graph_replays():
    from estorch_b200.backend import CudaBackend
    fresh = CudaBackend(torch.device("cuda", 0))
    dims, B, pairs = [32, 2048, 2048, 4], 128, 8
    n, table, theta, obs, tgt, offs = _problem(dims, B, pairs, 0, seed=5)
    d = Dev(fresh, theta, table, obs, tgt)
    of = dev(fresh, offs)
    ret = fresh.zeros(2 * pairs)

    def call(dd, dims_):
        fresh.eval_mlp(dims_, dd.th, dd.tb, of, None, pairs, 0.02, dd.ob, dd.tg, ret[:pairs], ret[pairs:],
                       precision="f16_any", table16=dd.tb16)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match=r"estk_status -4\).*captured"):
        with torch.cuda.graph(graph):
            call(d, dims)
    torch.cuda.synchronize()
    call(d, dims)                                         # eagerly it grows
    torch.cuda.synchronize()
    eager = ret.cpu().numpy().copy()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call(d, dims)
    # a wider shape grows the slab again; the graph captured before keeps the buffers it was captured with
    wide = [32, 4096, 4096, 4]
    _, table2, theta2, obs2, tgt2, _ = _problem(wide, B, pairs, 0, seed=6)
    call(Dev(fresh, theta2, table2, obs2, tgt2), wide)
    torch.cuda.synchronize()
    ret.zero_()
    graph.replay()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(ret.cpu().numpy(), eager)
    want, _ = _oracle(dims, theta, table, offs[:1], 0.02, obs, tgt, 0, 0, 0, "f16")
    assert rel_err(eager[[0, pairs]], want) < 1e-5


# ------------------------------------------------------------------ selection and the launch counter
def _fresh_process(code, *args):
    """Run `code` in a new interpreter (a profiling session there is the process's first: after one session
    has torn CUPTI down, a later one in the same process may record nothing) and return its last JSON line."""
    tests = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", code, *args, os.path.dirname(tests), tests],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("dims,B,kernels", [([320, 64, 32], 256, [SPLIT, STREAM]), ([64, 256, 64], 255, [SPLIT, STREAM]),
                                            ([64, 256, 64], 256, [CLUSTER]), ([784, 256, 10], 100, [SPLIT, STREAM])])
def test_kernel_selection_by_name(dims, B, kernels):
    code = """if True:
        import json, sys
        sys.path[:0] = sys.argv[3:]
        import numpy as np, torch
        from torch.profiler import ProfilerActivity, profile
        from estorch_b200.backend import CudaBackend
        from test_eval_mlp_f16_any_gpu import Dev, _problem, _run
        be = CudaBackend(torch.device("cuda", 0))
        dims, B = json.loads(sys.argv[1]), int(sys.argv[2])
        n, table, theta, obs, tgt, offs = _problem(dims, B, 4, 0)
        d = Dev(be, theta, table, obs, tgt)
        want, _ = _run(be, dims, d, offs, 0.02, 0)       # workspace growth and module load outside the profile
        n0 = be.launches
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device="cuda").mul_(2.0)
            got, _ = _run(be, dims, d, offs, 0.02, 0)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        ours = [m for m in names if any(k in m for k in ("eval_mlp", "split_obs"))]
        print(json.dumps({"names": ours, "torch": len(names) - len(ours), "launches": be.launches - n0,
                          "same_bits": bool(np.array_equal(got, want))}))
    """
    out = _fresh_process(code, json.dumps(dims), str(B))
    assert out["torch"] >= 1, out                        # the window recorded GPU activity
    assert out["same_bits"]
    assert len(out["names"]) == len(kernels) == out["launches"], out
    for name, k in zip(out["names"], kernels):
        assert f"::{k}" in name, out


def test_launch_counter_matches_profiled_kernels_in_fused_generations():
    code = """if True:
        import glob, json, os, re, sys
        sys.path[:0] = sys.argv[1:]
        os.environ["ESTORCH_B200_GRAPH"] = "0"
        import numpy as np, torch
        import estorch_b200 as E
        from _xent_oracle import MLP
        root = sys.argv[1]
        names = set()
        for path in glob.glob(os.path.join(root, "estorch_b200", "csrc", "*.cu")):
            names |= set(re.findall(r"__global__\\s+void\\s+(?:__launch_bounds__\\([^)]*\\)\\s*)?(\\w+)", open(path).read()))
        rng = np.random.RandomState(3)
        obs = torch.from_numpy(rng.standard_normal((100, 784)).astype(np.float32))
        tgt = torch.from_numpy(np.eye(10, dtype=np.float32)[rng.randint(0, 10, 100)])
        es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.02,
                  policy_kwargs={"dims": [784, 256, 10]}, agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy"),
                  optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 20, log_interval=4, eval_precision="f16")
        assert es._fused and es._precision == "f16_any"
        es.log = lambda: None
        es.train(n_steps=1)
        torch.cuda.synchronize()
        n0 = es._be.launches
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            es.train(n_steps=3)
            torch.cuda.synchronize()
        ks = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
              and any(k in e.name for k in names)]
        print(json.dumps({"kernels": len(ks), "launches": es._be.launches - n0,
                          "stream": sum("eval_mlp_tc_stream_kernel" in k for k in ks)}))
    """
    out = _fresh_process(code)
    assert out["kernels"] == out["launches"] > 0, out
    assert out["stream"] >= 3, out


# ------------------------------------------------------------------ public API
def _xent_es(dims, B, eval_precision, graph, monkeypatch, seed=2):
    monkeypatch.setenv("ESTORCH_B200_GRAPH", graph)
    rng = np.random.RandomState(seed)
    obs = torch.from_numpy(rng.standard_normal((B, dims[0])).astype(np.float32))
    tgt = torch.from_numpy(np.eye(dims[-1], dtype=np.float32)[rng.randint(0, dims[-1], B)])
    rec = []

    class R(E.ES):
        def log(self):
            rec.append((self.population_returns.copy(), self.episode_reward,
                        self._slots[0].theta.detach().cpu().numpy().copy()))
    torch.manual_seed(6)
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.02, policy_kwargs={"dims": dims},
           agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy"), optimizer_kwargs={"lr": 0.01},
           noise_table_size=1 << 20, eval_precision=eval_precision)
    return es, rec


def test_es_xent_classifier_f16_trains_fused_close_to_fp32_and_graph_equals_eager(monkeypatch):
    dims, B = [784, 256, 10], 256
    es, rec = _xent_es(dims, B, "f16", "0", monkeypatch)
    assert es._fused and es._precision == "f16_any"
    es.train(n_steps=3)
    ref, rref = _xent_es(dims, B, "fp32", "0", monkeypatch)
    assert ref._precision == "fp32"
    ref.train(n_steps=3)
    assert rel_err(rec[0][0], rref[0][0]) < 3e-5
    for gen in range(3):
        # ranks may swap between returns closer than the two evaluations' difference; Adam moves an entry
        # by at most lr per generation
        assert np.abs(rec[gen][2] - rref[gen][2]).max() <= 2 * 0.01 * (gen + 1) + 1e-6
        assert np.all(np.isfinite(rec[gen][0])) and np.isfinite(rec[gen][1])
    g, rg = _xent_es(dims, B, "f16", "1", monkeypatch)
    g.train(n_steps=5)
    e, re_ = _xent_es(dims, B, "f16", "0", monkeypatch)
    e.train(n_steps=5)
    assert sum(isinstance(v, tuple) for v in g.__dict__.get("_graphs", {}).values()) >= 1
    for a, b in zip(rg, re_):
        np.testing.assert_array_equal(a[0], b[0])
        np.testing.assert_array_equal(a[2], b[2])
        assert a[1] == b[1]
    # "auto" keeps the fp32 kernel on this shape
    auto, _ = _xent_es(dims, B, "auto", "0", monkeypatch)
    assert auto._precision == "fp32"


def _golden_es(g, graph, monkeypatch):
    monkeypatch.setenv("ESTORCH_B200_GRAPH", graph)
    rec = []

    class R(E.ES):
        def log(self):
            rec.append((self.population_returns.copy(), self.episode_reward))
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.1,
           policy_kwargs={"dims": [int(x) for x in g["dims"]]},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]), loss="cross_entropy"),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]),
           eval_precision="f16")
    assert es._fused and es._precision == "f16_any"
    es._table.copy_(torch.from_numpy(orc.round_f16(g["table"])))     # "f16" reads an exact fp16 table
    _set_theta(es.policy, g["theta0"])
    es.train(n_steps=3)
    return rec


def test_es_xent_golden_f16_any_with_and_without_graphs(monkeypatch):
    g = load_golden("es_xent_p64.npz")
    rec = _golden_es(g, "0", monkeypatch)
    # the golden table rounded to fp16 moves every member by sigma * 2^-12 * |t| at most, less than the fp16
    # rounding of the weights themselves
    for gen in range(3):
        print(f"gen {gen}: returns vs golden {rel_err(rec[gen][0][:, 0], g['returns'][gen][:, 0]):.2e}")
        assert rel_err(rec[gen][0][:, 0], g["returns"][gen][:, 0]) < 1e-4
        assert abs(rec[gen][1] - float(g["episode_reward"][gen])) < 1e-4 * abs(float(g["episode_reward"][gen]))
    for a, b in zip(_golden_es(g, "1", monkeypatch), rec):
        np.testing.assert_array_equal(a[0], b[0])
        assert a[1] == b[1]


def test_nsr_xent_golden_f16_any():
    g = load_golden("nsr_xent_p32.npz")
    rec = []

    class R(E.NSR_ES):
        def log(self):
            rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward, idx=self.idx))
    np.random.seed(123)
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=32, sigma=0.02,
           policy_kwargs={"dims": [int(x) for x in g["dims"]]},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]), bc_obs=64,
                             bc_dim=256, loss="cross_entropy"),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]),
           eval_precision="f16")
    assert es._fused and es._precision == "f16_any"
    es._table.copy_(torch.from_numpy(orc.round_f16(g["table"])))
    for i, (p, _) in enumerate(es.meta_population):
        _set_theta(p, g["meta_theta0"][i])
        es._slots[i].push_theta()
    es._archive = [a.copy() for a in g["archive0"]]
    np.random.seed(123)
    es.train(n_steps=len(g["grad"]))
    # generation 0 evaluates the golden's members; from its update on, ranks may swap between returns closer
    # than the f16 evaluate's distance from fp32, and the post-update rollout sees a slightly different theta
    assert rel_err(rec[0]["returns"][:, 0], g["returns"][0][:, 0]) < 3e-5
    for gen in range(len(g["grad"])):
        ep = float(g["episode_reward"][gen])
        print(f"gen {gen}: returns vs golden {rel_err(rec[gen]['returns'][:, 0], g['returns'][gen][:, 0]):.2e}, "
              f"episode {abs(rec[gen]['episode'] - ep) / abs(ep):.2e}")
        assert rec[gen]["idx"] == int(g["idx"][gen])
        assert rel_err(rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 5e-4   # the drift compounds
        # the novelty is a kNN distance between behaviour characteristics, the logits, which f16 reproduces to
        # the 2e-3 of the BC checks above; the archive then holds the drifting centres' BCs
        assert rel_err(rec[gen]["returns"][:, 1], g["returns"][gen][:, 1]) < (5e-3 if gen == 0 else 2e-2)
        assert abs(rec[gen]["episode"] - ep) < 5e-4 * abs(ep)


def test_nsr_es_with_bc_trains_fused_f16_any():
    rng = np.random.RandomState(5)
    dims, B = [24, 64, 64, 4], 256
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
           noise_table_size=1 << 20, eval_precision="f16")
    assert es._fused and es._be.name == "cuda" and es._precision == "f16_any"
    es.train(n_steps=3)
    assert len(rec) == 3
    for r, ep in rec:
        assert np.all(np.isfinite(r)) and np.isfinite(ep)
