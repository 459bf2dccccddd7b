"""The TF32 convolutional evaluate (estk_eval_cnn_tf32, estk_eval_cnn_tf32.cu) on the H100: its rounding pinned
through the public entry, every code and every test shape against the TF32 rounding model and the float64
forward of the fp32 rows, prediction flips of the accuracy against the fp32 kernel, bit-exact identities
(materialised rows, sigma = 0, repeats with and without order, CUDA-graph replay), the slab within its workspace
bound, and ES training in the mode.

Bounds.  Against the rounding model (tests/_cnn_tf32_oracle.py: the same rounded operands, float64 sums) every
output is held to its own bound from ``forward_tf32_bounds``: its layer's fp32 accumulation, 2 (K + 2) 2^-24
times the sum of |terms|, plus one TF32 spacing times |w| for every input that lies within its error bound of a
TF32 rounding boundary (an operand-rounding flip) -- the outputs such a flip can reach are counted and
reported.  Every output is also held to BAR_MODEL = u = 2^-11 (max-norm relative).  Against the float64 forward of
the fp32 weights each layer rounds two operands (u/2 each), so outputs and returns are held to 2 * n_layers * u
(max-norm relative)."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA GPU", allow_module_level=True)

from estorch_b200 import ES, NSR_ES, DeviceAgent, _capi  # noqa: E402
from estorch_b200.backend import CudaBackend, cnn_desc  # noqa: E402
from _cnn_oracle import HIDDEN, image_task, pack, param_count, policy_class  # noqa: E402
from _cnn_tf32_oracle import LOSS_ACCURACY, forward_tf32, forward_tf32_bounds, returns64, rna_tf32  # noqa: E402

XENT, TANH = _capi.ESTK_LOSS_XENT, _capi.ESTK_ACT_OUT_TANH
U = 2.0 ** -11
BAR_MODEL = U
SIGMA = 0.05
# (input shape, convs (out_c, k, stride, pad), linear widths, B, pairs): tests/test_cnn_gpu.py's CASES
CASES = {
    "mnist": ((1, 28, 28), [(16, 5, 2, 2), (32, 5, 2, 2)], [10], 32, 64),
    "c3_k3_p1": ((3, 11, 9), [(7, 3, 1, 1)], [5], 3, 3),
    "k8_s4_then_1x1": ((3, 16, 16), [(7, 8, 4, 0), (3, 1, 1, 0)], [12, 4], 1, 1),
    "four_convs": ((2, 13, 13), [(3, 3, 2, 2), (7, 3, 1, 0), (5, 1, 1, 0), (4, 3, 1, 1)], [9, 6, 2], 257, 8),
    "minatar": ((6, 10, 10), [(16, 3, 1, 0)], [128, 4], 32, 1024),
    "atari_small": ((4, 36, 36), [(16, 8, 4, 0), (32, 4, 2, 0)], [64, 6], 5, 64),
    "k5_p2_odd": ((3, 7, 7), [(3, 5, 1, 2)], [3], 3, 1),
    "slab_3x128x128": ((3, 128, 128), [(32, 3, 1, 1), (4, 8, 8, 0)], [4], 2, 2),
}
LOSSES = (0, TANH, XENT, LOSS_ACCURACY)


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _code(n_conv, hidden=0, rest=0):
    return hidden | rest | n_conv << 24


def _setup(be, dims, code, pairs, seed=0, scale=1.0):
    torch.manual_seed(seed)
    pol = policy_class(code >> 24, HIDDEN[code & 0xff], bool(code & TANH))(dims)
    theta = torch.nn.utils.parameters_to_vector(pol.parameters()).detach().to(be.device).contiguous() * scale
    n = theta.numel()
    assert n == param_count(dims, code >> 24)
    table = be.alloc(max(1 << 16, (n + 31) // 32 * 32 + 32 * 4096))
    be.fill_noise_table(table, 11 + seed)
    offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
    be.make_offsets(5 + seed, None, 0, 0, pairs, table.numel(), n, offsets, order)
    return theta, table, offsets, order


def _data(shape, B, out, classes, seed=1):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(B, *shape, generator=g)
    if classes:
        tgt = torch.nn.functional.one_hot(torch.randint(0, out, (B,), generator=g), out).float()
    else:
        tgt = torch.rand(B, out, generator=g) * 1.6 - 0.8
    return obs, tgt


def _eval(be, dims, code, theta, table, offsets, order, pairs, sigma, obs, tgt, precision="tf32"):
    """Returns [2*pairs] and every member's outputs [2*pairs, B, out] (read through the BC)."""
    B, out = tgt.shape
    ret, bc = be.zeros(2 * pairs), be.zeros(2 * pairs, B * out)
    be.eval_cnn(dims, theta, table, offsets, order, pairs, sigma, obs, tgt, ret[:pairs], ret[pairs:], bc[:pairs],
                bc[pairs:], B, B * out, act=code, precision=precision)
    torch.cuda.synchronize()
    return ret, bc.view(2 * pairs, B, out)


def _rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _check(be, name, hidden, rest):
    shape, convs, linears, B, pairs = CASES[name]
    dims, code = pack(shape, convs, linears), _code(len(convs), hidden, rest)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, linears[-1], bool(rest & (XENT | LOSS_ACCURACY))))
    ret, y = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    rows = be.alloc(2 * pairs, theta.numel())
    be.perturb_rows(theta, table, offsets, pairs, SIGMA, 0, 2 * pairs, rows)
    R, X, T = rows.cpu().numpy(), obs.cpu().numpy(), tgt.cpu().numpy()
    model = [forward_tf32_bounds(r, dims, code, X) for r in R]
    y_model, bound, exposed = (np.stack(t) for t in zip(*model))
    y_64 = np.stack([_forward64(r, dims, code, X) for r in R])
    yk = y.cpu().numpy()
    err = np.abs(yk - y_model)
    e_model, e_64 = _rel(yk, y_model), _rel(yk, y_64)
    bar64 = 2 * (len(convs) + len(linears)) * U
    worst = float((err / np.maximum(bound, 1e-300)).max())
    print(f"{name} code={code:#x}: outputs vs model {e_model:.2e}, worst error / own bound {worst:.2f}; "
          f"{int(exposed.sum())} of {yk.size} reachable by an operand-rounding flip; vs float64 {e_64:.2e} "
          f"(bound {bar64:.1e})")
    assert (err <= bound).all(), worst
    assert e_model <= BAR_MODEL and e_64 <= bar64
    if not rest & LOSS_ACCURACY:
        r64 = returns64(y_64, T, code)
        e_r = _rel(ret.cpu().numpy(), r64)
        print(f"   returns vs float64 {e_r:.2e}")
        assert e_r <= bar64


def _forward64(row, dims, code, X):
    """The float64 forward of the member's fp32 weights (no operand rounding)."""
    from _cnn_oracle import forward
    return forward(row, dims, code, X, dt=np.float64)


def test_rounding_pinned_through_the_public_entry(be):
    """1x1x1 images, conv 1->1 k1, ReLU, Linear 1->1: y = rna(w1) * rna(relu(rna(w0) * rna(x) + b0)) + b1, each
    product of two TF32 operands exact in fp32, so the outputs equal the restatement bit for bit."""
    dims, code = pack((1, 1, 1), [(1, 1, 1, 0)], [1]), _code(1)
    tie, ulp = 2.0 ** -11, 2.0 ** -23
    xs = np.array([1 + tie, 1 + tie - ulp, 1 + tie + ulp, 1 + 3 * tie, 1.5 + tie, 3 - tie, 0.75 + tie / 2, 2 + 2 * tie,
                   1 + 5 * tie - ulp, 7 + 7 * 4 * tie], np.float32)
    for w0, b0, w1, b1 in [(1 + tie, 0.0, 1 + 3 * tie, 0.0), (1 + tie - ulp, 0.25, 1.0 + tie + ulp, -0.5),
                           (0.5 + tie / 2, 2.0 ** -20, 3 + 3 * tie, 1.0 + ulp)]:
        theta = torch.tensor([w0, b0, w1, b1], dtype=torch.float32, device=be.device)
        B = xs.size
        obs = torch.from_numpy(xs).reshape(B, 1, 1, 1).to(be.device)
        tgt = be.zeros(B, 1)
        ret, bc = be.zeros(1), be.zeros(B)
        be.eval_cnn_center(dims, theta, obs, tgt, ret, bc, B, B, precision="tf32", act=code)
        torch.cuda.synchronize()
        p = np.float32
        h = np.maximum(rna_tf32(p(w0)) * rna_tf32(xs) + p(b0), p(0))
        want = (rna_tf32(p(w1)) * rna_tf32(h) + p(b1)).astype(np.float32)
        assert np.array_equal(bc.cpu().numpy().view(np.uint32), want.view(np.uint32)), (bc.cpu().numpy(), want)


@pytest.mark.parametrize("hidden", list(HIDDEN))
@pytest.mark.parametrize("rest", LOSSES)
def test_every_code_against_model_and_float64(be, hidden, rest):
    _check(be, "c3_k3_p1", hidden, rest)


@pytest.mark.parametrize("name", [n for n in CASES if n != "c3_k3_p1"])
def test_shapes_against_model_and_float64(be, name):
    i = list(CASES).index(name)
    _check(be, name, list(HIDDEN)[i % 5], LOSSES[i % 4])


def test_accuracy_prediction_flips_against_fp32(be):
    shape, convs, linears, B, pairs = CASES["mnist"]
    dims, code = pack(shape, convs, linears), _code(2, 0, LOSS_ACCURACY)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, 10, True))
    r32, y32 = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt, precision="fp32")
    rtf, ytf = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    flips = int((y32.argmax(-1) != ytf.argmax(-1)).sum())
    print(f"accuracy: {flips} prediction flips of {y32.shape[0] * y32.shape[1]}, max return change "
          f"{float((r32 - rtf).abs().max()):.3e}")
    assert flips <= 0.01 * y32.shape[0] * y32.shape[1]


def test_identities(be):
    """A member is its materialised row through the centre form; sigma = 0 gives every member the centre's bits;
    repeats with and without order give the same bits."""
    for name in ("mnist", "four_convs", "minatar"):
        shape, convs, linears, B, pairs = CASES[name]
        pairs = min(pairs, 8)
        dims, code = pack(shape, convs, linears), _code(len(convs), 4, XENT)
        theta, table, offsets, order = _setup(be, dims, code, pairs)
        obs, tgt = (t.to(be.device) for t in _data(shape, B, linears[-1], True))
        ret, y = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
        rows = be.alloc(2 * pairs, theta.numel())
        be.perturb_rows(theta, table, offsets, pairs, SIGMA, 0, 2 * pairs, rows)
        out = tgt.shape[1]
        for m in (0, pairs - 1, pairs, 2 * pairs - 1):
            r1, b1 = be.zeros(1), be.zeros(B * out)
            be.eval_cnn_center(dims, rows[m].contiguous(), obs, tgt, r1, b1, B, B * out, precision="tf32", act=code)
            torch.cuda.synchronize()
            assert torch.equal(r1[0], ret[m]) and torch.equal(b1.view(B, out), y[m]), (name, m)
        r2, y2 = _eval(be, dims, code, theta, table, offsets, None, pairs, SIGMA, obs, tgt)
        r3, y3 = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
        assert torch.equal(r2, ret) and torch.equal(y2, y) and torch.equal(r3, ret) and torch.equal(y3, y)
        r0, y0 = _eval(be, dims, code, theta, table, offsets, order, pairs, 0.0, obs, tgt)
        rc, bcc = be.zeros(1), be.zeros(B * out)
        be.eval_cnn_center(dims, theta, obs, tgt, rc, bcc, B, B * out, precision="tf32", act=code)
        torch.cuda.synchronize()
        assert torch.equal(r0, rc.expand(2 * pairs)) and torch.equal(y0, bcc.view(1, B, out).expand_as(y0))


def test_graph_replay_equals_eager(be):
    shape, convs, linears, B, pairs = CASES["atari_small"]
    dims, code = pack(shape, convs, linears), _code(2, 0, 0)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, linears[-1], False))
    ret_e, y_e = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    ret, bc = be.zeros(2 * pairs), be.zeros(2 * pairs, B * linears[-1])
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            be.eval_cnn(dims, theta, table, offsets, order, pairs, SIGMA, obs, tgt, ret[:pairs], ret[pairs:],
                        bc[:pairs], bc[pairs:], B, B * linears[-1], act=code, precision="tf32")
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(ret, ret_e) and torch.equal(bc.view_as(y_e), y_e)


def test_refusals_and_supported(be):
    dims, code = pack((1, 28, 28), [(16, 5, 2, 2)], [10]), _code(1, 0, XENT)
    d = cnn_desc(dims, code)
    lib = be.lib
    assert lib.estk_eval_cnn_tf32_supported(C_ref(d), 256) == 1
    for bad in (_capi.ESTK_ACTIONS, _capi.ESTK_CELL_GRU, 2 << 16):
        d2 = cnn_desc(dims, (1 << 24) | bad)
        assert lib.estk_eval_cnn_tf32_supported(C_ref(d2), 256) == 0
    with pytest.raises(RuntimeError, match="estk_status -1"):
        x = be.zeros(4, 1, 28, 28)
        be.eval_cnn(dims, be.zeros(100), None, None, None, 1, 0.0, x, be.zeros(4, 10), be.zeros(1), None,
                    act=(1 << 24) | _capi.ESTK_ACTIONS, precision="tf32")


def C_ref(d):
    import ctypes
    return ctypes.byref(d)


def _classifier_es(precision, cls=ES, P=64, batch_size=None, **kw):
    obs, tgt = image_task(256, (1, 12, 12), 4, seed=0)
    dims = pack((1, 12, 12), [(8, 3, 2, 1)], [4])
    torch.manual_seed(0)
    agent_kw = dict(obs=obs, target=tgt, loss="cross_entropy")
    if batch_size:
        agent_kw["batch_size"] = batch_size
    es = cls(lambda: policy_class(1)(dims), DeviceAgent, torch.optim.Adam, population_size=P, sigma=0.05,
             agent_kwargs=agent_kw, optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 20,
             eval_precision=precision, **kw)
    es.log = lambda: None
    return es, obs, tgt


def test_example_cnn_classifier_learns_in_tf32():
    """examples/cnn_classifier.py at its test settings, evaluated in "tf32", clears the fp32 test's bar."""
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "cnn_classifier.py")
    spec = importlib.util.spec_from_file_location("cnn_classifier", path)
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    first, last, acc0, acc1 = ex.main(generations=ex.TEST_GENERATIONS, population=ex.TEST_POPULATION,
                                      eval_precision="tf32")
    print(f"cnn_classifier in tf32: centre return {first:.4f} -> {last:.4f}, accuracy {acc0:.3f} -> {acc1:.3f}")
    assert acc1 >= acc0 + ex.TEST_MARGIN


def test_nsr_cross_entropy_with_bc_runs_fused_in_tf32():
    obs, tgt = image_task(64, (1, 12, 12), 4, seed=0)
    dims = pack((1, 12, 12), [(8, 3, 2, 1)], [4])
    torch.manual_seed(0)
    es = NSR_ES(lambda: policy_class(1)(dims), DeviceAgent, torch.optim.Adam, population_size=32, sigma=0.05,
                agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy", bc_obs=2, bc_dim=8),
                optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 20, eval_precision="tf32")
    es.log = lambda: None
    assert es._fused and es._precision == "tf32"
    es.train(n_steps=3)
    assert np.isfinite(es.population_returns).all()


def test_batch_size_runs_fused_and_replays_from_a_graph(monkeypatch):
    """Minibatches in tf32: generations replayed from a CUDA graph leave exactly the state of eager launches."""
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ESTORCH_B200_GRAPH", mode)
        es, _, _ = _classifier_es("tf32", batch_size=64)
        assert es._fused and es._sampling and es._precision == "tf32"
        es.train(n_steps=6)
        torch.cuda.synchronize()
        graphs = sum(isinstance(v, tuple) for v in es.__dict__.get("_graphs", {}).values())
        out[mode] = (es._slots[0].theta.clone(), es.population_returns.copy(), graphs)
    assert out["1"][2] >= 1 and out["0"][2] == 0          # graphs were actually used / not used
    assert torch.equal(out["1"][0], out["0"][0])
    np.testing.assert_array_equal(out["1"][1], out["0"][1])
    assert np.isfinite(out["1"][1]).all()


def test_slab_shape_runs_within_the_workspace_bound():
    """3x512x512 with 16 channels at B = 2: one image per chunk, and the grid's slab capped at 1 GB (every resident
    CTA's slab would be ~8 GB); the outputs are within the bounds of the other shapes."""
    be2 = CudaBackend()
    shape, convs, linears, B, pairs = (3, 512, 512), [(16, 3, 1, 1), (4, 16, 16, 0)], [4], 2, 2
    dims, code = pack(shape, convs, linears), _code(2, 0, 0)
    theta, table, offsets, order = _setup(be2, dims, code, pairs)
    obs, tgt = (t.to(be2.device) for t in _data(shape, B, 4, False))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(be2.device)[0]
    ret, y = _eval(be2, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    grown = free0 - torch.cuda.mem_get_info(be2.device)[0]
    assert grown < (2 << 30), grown
    rows = be2.alloc(2 * pairs, theta.numel())
    be2.perturb_rows(theta, table, offsets, pairs, SIGMA, 0, 2 * pairs, rows)
    R, X = rows.cpu().numpy(), obs.cpu().numpy()
    y_64 = np.stack([_forward64(r, dims, code, X) for r in R])
    assert _rel(y.cpu().numpy(), y_64) <= 2 * 3 * U


def test_train_n_proc_2_keeps_theta_identical_across_ranks(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess
    import sys
    import textwrap
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "user_script.py"
    script.write_text(textwrap.dedent(f"""
        import os, sys, numpy as np, torch
        sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
        import estorch_b200 as E
        from _cnn_oracle import image_task, pack, policy_class
        obs, tgt = image_task(256, (1, 12, 12), 4, seed=0)
        dims = pack((1, 12, 12), [(8, 3, 2, 1)], [4])
        torch.manual_seed(0)
        es = E.ES(policy_class(1), E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.05,
                  policy_kwargs={{"dims": dims}}, agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy"),
                  optimizer_kwargs={{"lr": 0.03}}, noise_table_size=1 << 20, eval_precision="tf32")
        es.log = lambda: None
        es.train(n_steps=3, n_proc=2)
        torch.cuda.synchronize()
        assert es._precision == "tf32"
        np.save(os.path.join({str(tmp_path)!r}, f"theta_rank{{es.rank}}.npy"), es._slots[0].theta.cpu().numpy())
    """))
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    np.testing.assert_array_equal(np.load(tmp_path / "theta_rank0.npy"), np.load(tmp_path / "theta_rank1.npy"))


def test_resume_is_bit_identical_in_tf32(tmp_path):
    a, _, _ = _classifier_es("tf32")
    a.train(n_steps=3)
    path = str(tmp_path / "ck.pt")
    a.save_checkpoint(path) if hasattr(a, "save_checkpoint") else pytest.skip("no checkpoint API")
    a.train(n_steps=2)
    b, _, _ = _classifier_es("tf32")
    b.load_checkpoint(path)
    b.train(n_steps=2)
    assert torch.equal(a._slots[0].theta, b._slots[0].theta)


# ------------------------------------------------------------------ what ES consumes: the signal across sigma
SIG_PAIRS = 32
GRAD_BAR = 3e-2
SIG_SIGMAS = (0.05, 0.02, 5e-3, 1e-3, 2e-4)
SIG_CELLS = ([(s, w, 1.0) for s in SIG_SIGMAS for w in (1.0, 4.0, 8.0)] + [(5e-3, 4.0, 100.0)])


def tf32_in_domain(sigma, scale, obs_scale):
    """The documented accuracy domain of "tf32" (measured by the cells below): sigma >= 5e-3 with weights up to
    8x their initial scale, observations of any scale.  Below it the 11-bit operands reorder members: gradient
    rel-L2 up to 0.08 at sigma = 1e-3 and 0.33 at 2e-4 (8x init)."""
    return sigma >= 5e-3 and scale <= 8


@pytest.mark.parametrize("sigma,scale,obs_scale", SIG_CELLS)
def test_tf32_signal_vs_rounding_model_and_domain(be, sigma, scale, obs_scale):
    """The tf32 returns against the float64 returns of the fp32 rows, on what ES consumes (pair differences,
    ranks, the gradient), next to the TF32 rounding model's: the kernel adds no error beyond its model, the
    returns are within tau_tf32 (the per-return bound of _fp64_signal's construction with the TF32 unit), and
    inside the domain the gradient is within GRAD_BAR of the float64-return gradient."""
    import _fp64_signal as sig
    from _cnn_tf32_oracle import tau_tf32
    dims, code = pack((3, 12, 12), [(8, 3, 2, 1), (16, 3, 1, 0)], [16, 4]), 2 << 24
    B = 64
    torch.manual_seed(0)
    pol = policy_class(2)(dims)
    theta = (torch.nn.utils.parameters_to_vector(pol.parameters()).detach().numpy() * scale).astype(np.float32)
    n = theta.size
    table = be.alloc(max(1 << 16, (n + 31) // 32 * 32 + 32 * 16 * SIG_PAIRS))
    be.fill_noise_table(table, 7)
    offs, order = be.alloc(SIG_PAIRS, dtype=torch.int64), be.alloc(SIG_PAIRS, dtype=torch.int32)
    be.make_offsets(8, None, 0, 0, SIG_PAIRS, table.numel(), n, offs, order)
    g = np.random.RandomState(4)
    obs = (g.standard_normal((B, 3, 12, 12)) * obs_scale).astype(np.float32)
    tgt = g.standard_normal((B, 4)).astype(np.float32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(be.device)
    th_d = dev(theta)
    ret = be.zeros(2 * SIG_PAIRS)
    be.eval_cnn(dims, th_d, table, offs, order, SIG_PAIRS, sigma, dev(obs), dev(tgt), ret[:SIG_PAIRS],
                ret[SIG_PAIRS:], act=code, precision="tf32")
    rows = sig.members(theta, table.cpu().numpy(), offs.cpu().numpy(), sigma)
    r64, _ = sig.cnn_reference(rows, dims, code, obs, tgt)
    y64 = np.stack([_forward64(r, dims, code, obs) for r in rows])
    tau = tau_tf32(y64, tgt, 3)
    r_model = returns64(np.stack([forward_tf32(r, dims, code, obs) for r in rows]), tgt, code)
    _, g64 = sig.device_gradient(be, dev(r64.astype(np.float32)), table, offs, order, th_d)
    _, gk = sig.device_gradient(be, ret, table, offs, order, th_d)
    _, gm = sig.device_gradient(be, dev(r_model.astype(np.float32)), table, offs, order, th_d)
    r = ret.cpu().numpy()
    m = sig.signal_metrics(r, r64, gk, g64)
    mm = sig.signal_metrics(r_model, r64, gm, g64)
    d64 = r64[:SIG_PAIRS] - r64[SIG_PAIRS:]
    kernel_vs_model = float(np.max(np.abs((r[:SIG_PAIRS] - r[SIG_PAIRS:]) - (r_model[:SIG_PAIRS] -
                                                                              r_model[SIG_PAIRS:]))) / d64.std())
    domain = tf32_in_domain(sigma, scale, obs_scale)
    cell = dict(mode="tf32", sigma=sigma, scale=scale, obs_scale=obs_scale, in_domain=domain, kernel=m, model=mm,
                diff_kernel_vs_model_over_std=kernel_vs_model, err_over_tau=float(np.max(np.abs(r - r64) / tau)))
    print("SIGNAL_FIDELITY_TF32 " + json.dumps(cell, sort_keys=True))
    assert np.all(np.abs(r - r64) <= tau), cell
    # the kernel adds no error beyond its rounding model
    assert kernel_vs_model < 0.1, cell
    assert m["returns_max_rel"] <= 2 * mm["returns_max_rel"] + 1e-6, cell
    assert m["diff_wrong_sign"] <= 2 * mm["diff_wrong_sign"] + 2 / SIG_PAIRS, cell
    assert m["grad_rel_l2"] <= 2 * mm["grad_rel_l2"] + 1.5e-2, cell
    if domain:
        assert m["grad_rel_l2"] <= GRAD_BAR, cell
