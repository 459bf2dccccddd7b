"""Classification accuracy (include/estk.h ESTK_LOSS_ACCURACY) on the H100: in every MLP evaluate mode (fp32
shared-memory and streamed, f16 / bf16 / bf16s cluster, f16_any streamed) and in the convolutional evaluate, every
member's return is exactly count / B of its own logits (read back as the behaviour characteristic with bc_obs = B);
engineered ties and NaN logits follow torch.argmax; the fp32 count against a float64 forward; prediction flips of
the 16-bit modes against fp32; the reference goldens; graph replay; and one learning run on minibatches."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import es_oracle as orc
import _accuracy_oracle as ao
from _cnn_oracle import pack, param_count as cnn_param_count
from test_eval_mlp_act_gpu import _eval, _tc_problem, dev

pytestmark = pytest.mark.gpu
ACC = ao.LOSS_ACCURACY
HIDDEN = (0, 1, 3, 4, 5)                       # ReLU, Tanh, ELU, SiLU, LeakyReLU


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def _labels_target(rng, B, C, soft=False):
    lab = rng.randint(0, C, B)
    if not soft:
        return np.eye(C, dtype=np.float32)[lab]
    t = rng.dirichlet(np.ones(C), B).astype(np.float32)
    t[np.arange(B), lab] += 1.0
    return t


def _tc_kw(be, mode, theta, table):
    kw = {}
    if mode in ("f16", "f16_any"):
        kw["table16"] = be.alloc(table.size, dtype=torch.float16)
        assert be.shadow_f16(dev(be, table), kw["table16"]) == 0
    elif mode == "bf16s":
        kw["theta16"] = be.alloc(theta.size, dtype=torch.bfloat16)
        kw["table16"] = be.alloc(table.size, dtype=torch.bfloat16)
        be.shadow_bf16(dev(be, theta), kw["theta16"])
        be.shadow_bf16(dev(be, table), kw["table16"])
    return kw


def _want(logits, tgt):
    """count / B of each member's logits [M, B*C] under torch.argmax's rule, fp32."""
    B, C = tgt.shape
    y = torch.from_numpy(logits.reshape(-1, B, C))
    lab = torch.from_numpy(tgt).argmax(1)
    cnt = (y.argmax(2) == lab).sum(1).numpy()
    return (cnt.astype(np.float32) / np.float32(B)).astype(np.float32)


def _check_counts(be, dims, B, pairs, mode, code, theta, table, offs, obs, tgt, sigma=0.02):
    C = dims[-1]
    kw = _tc_kw(be, mode, theta, table)
    ret, logits, _ = _eval(be, dims, theta, table, offs, sigma, obs, tgt, code | ACC, B, B * C, precision=mode, **kw)
    want = _want(logits, tgt)
    np.testing.assert_array_equal(ret, want)
    assert ret.tobytes() == want.tobytes()              # +0.0 for no correct row, never -0.0
    return ret, logits


# (mode, dims, B, pairs): every kernel and the batch sizes around its chunking
CASES = [("fp32", [20, 64, 10], 1, 3), ("fp32", [20, 64, 10], 100, 3), ("fp32", [20, 64, 10], 256, 3),
         ("fp32", [20, 64, 10], 257, 2), ("fp32", [784, 256, 10], 60000, 1), ("fp32", [20, 64, 10], 64, 1024),
         ("f16", [64, 128, 256], 256, 3), ("f16", [128, 512, 512, 512, 512, 256], 512, 2),
         ("bf16", [64, 128, 256], 256, 3), ("bf16s", [64, 128, 256], 256, 3), ("f16", [64, 64, 32], 256, 1024),
         ("f16_any", [784, 256, 10], 1, 3), ("f16_any", [784, 256, 10], 100, 3), ("f16_any", [33, 70, 10], 257, 2)]


@pytest.mark.parametrize("code", HIDDEN)
@pytest.mark.parametrize("mode,dims,B,pairs", CASES)
def test_every_return_is_the_count_of_the_kernels_own_logits(be, mode, dims, B, pairs, code):
    if mode in ("f16", "bf16", "bf16s"):
        assert be.eval_supports_f16(dims, B, act=code | ACC) and be.eval_supports_bf16(dims, B, act=code | ACC)
    if mode == "f16_any":
        assert not be.eval_supports_f16(dims, B, act=code | ACC) and be.eval_supports_f16_any(dims, B, act=code | ACC)
    n, table, theta, obs, _, offs = _tc_problem(dims, B, pairs)
    tgt = _labels_target(np.random.RandomState(B + code), B, dims[-1], soft=code % 2 == 1)
    ret, _ = _check_counts(be, dims, B, pairs, mode, code, theta, table, offs, obs, tgt)
    assert len(np.unique(ret)) > 1 or B == 1
    # the centre form: theta itself
    one, bc = be.zeros(1), be.zeros(B * dims[-1])
    be.eval_mlp_center(dims, dev(be, theta), dev(be, obs), dev(be, tgt), one, bc, B, B * dims[-1],
                       precision=mode, act=code | ACC, **({"theta16": _tc_kw(be, mode, theta, table)["theta16"]}
                                                          if mode == "bf16s" else {}))
    assert float(one) == float(_want(bc.cpu().numpy()[None], tgt)[0])


def _engineered(dims, B, seed=5):
    """A theta whose last layer has zero weights, so every logit row is the bias: ties at two columns far apart
    (possibly in different threads, column blocks and N tiles), and a second bias with two NaN columns."""
    rng = np.random.RandomState(seed)
    n, table, theta, obs, _, offs = _tc_problem(dims, B, 2, seed)
    C, K = dims[-1], dims[-2]
    wlast = n - C - C * K
    theta[wlast:n - C] = 0.0
    lo, hi = 1, C - 2
    bias = np.full(C, -1.0, np.float32)
    bias[[lo, hi]] = 3.0
    nan = bias.copy()
    nan[[hi - 1 if hi - 1 > lo else hi, lo + 1 if lo + 1 < C else lo]] = np.nan
    lab = rng.choice([lo, hi, 0], B)
    tgt = np.eye(C, dtype=np.float32)[lab]
    return n, table, theta, obs, offs, tgt, bias, nan


@pytest.mark.parametrize("mode,dims,B", [("fp32", [20, 64, 10], 100), ("fp32", [784, 256, 10], 3000),
                                         ("f16", [64, 128, 256], 256), ("bf16", [64, 128, 256], 256),
                                         ("bf16s", [64, 128, 256], 256), ("f16_any", [784, 256, 10], 100),
                                         ("f16_any", [40, 64, 300], 70)])
def test_ties_and_nans_follow_torch_argmax(be, mode, dims, B):
    n, table, theta, obs, offs, tgt, bias, nan = _engineered(dims, B)
    for b in (bias, nan):
        th = theta.copy()
        th[n - dims[-1]:] = b
        # sigma = 0: every member has exactly these logits (and the bf16 shadows round -1 and 3 exactly)
        ret, logits = _check_counts(be, dims, B, len(offs), mode, 0, th, table, offs, obs, tgt, sigma=0.0)
        y = logits.reshape(-1, B, dims[-1])
        pred = torch.from_numpy(y).argmax(2)
        assert bool((pred == int(np.argmax(b))).all())     # the first of the tied (or NaN) columns


def test_cnn_returns_are_the_count_of_its_logits(be):
    dims = pack((2, 10, 10), [(6, 3, 1, 1), (8, 3, 2, 0)], [16, 7])
    n = cnn_param_count(dims, 2)
    rng = np.random.RandomState(3)
    for B, pairs in ((1, 3), (100, 3), (257, 2)):
        theta = (rng.standard_normal(n) * 0.3).astype(np.float32)
        table = rng.standard_normal(n + 4096).astype(np.float32)
        offs = orc.noise_offsets(2, 0, 0, pairs, table.size, n)
        obs = rng.standard_normal((B, 2, 10, 10)).astype(np.float32)
        tgt = _labels_target(rng, B, 7)
        for code in HIDDEN:
            act = 2 << 24 | code | ACC
            ret, bp, bm = be.zeros(2 * pairs), be.zeros(pairs, B * 7), be.zeros(pairs, B * 7)
            order = dev(be, np.arange(pairs, dtype=np.int32))
            be.eval_cnn(dims, dev(be, theta), dev(be, table), dev(be, offs), order, pairs, 0.05, dev(be, obs),
                        dev(be, tgt), ret[:pairs], ret[pairs:], bp, bm, B, B * 7, act=act)
            logits = torch.cat([bp, bm]).cpu().numpy()
            np.testing.assert_array_equal(ret.cpu().numpy(), _want(logits, tgt))
        # a NaN and a tie through the head's bias, sigma = 0
        th = theta.copy()
        th[n - 7 - 7 * 16:n - 7] = 0.0
        th[n - 7:] = [-1, 2, 0, 2, np.nan, 1, np.nan]
        ret, bp, bm = be.zeros(2 * pairs), be.zeros(pairs, B * 7), be.zeros(pairs, B * 7)
        be.eval_cnn(dims, dev(be, th), dev(be, table), dev(be, offs), order, pairs, 0.0, dev(be, obs), dev(be, tgt),
                    ret[:pairs], ret[pairs:], bp, bm, B, B * 7, act=2 << 24 | ACC)
        np.testing.assert_array_equal(ret.cpu().numpy(), _want(torch.cat([bp, bm]).cpu().numpy(), tgt))
        assert ret.cpu().numpy()[0] == np.float32(np.float32((tgt.argmax(1) == 4).sum()) / np.float32(B))


# ------------------------------------------------------------------ against float64, and the 16-bit modes
MARGIN = 1e-5          # relative gap between the top two float64 logits below which fp32 may order them otherwise


@pytest.mark.parametrize("dims,B", [([784, 256, 10], 4096), ([128, 512, 512, 512, 512, 256], 512)])
def test_fp32_count_against_float64_and_flips_of_the_16_bit_modes(be, dims, B):
    pairs = 8
    n, table, theta, obs, _, offs = _tc_problem(dims, B, pairs)
    tgt = _labels_target(np.random.RandomState(1), B, dims[-1])
    ret32, y32, _ = _eval(be, dims, theta, table, offs, 0.02, obs, tgt, ACC, B, B * dims[-1])
    pop, _ = orc.sample_population(theta, table, offs, 0.02)
    lab = tgt.argmax(1)
    near = 0
    for m in range(2 * pairs):
        layers = orc.mlp_unflatten(pop[m].astype(np.float64), dims)
        h = obs.astype(np.float64)
        for i, (w, b) in enumerate(layers):
            h = h @ w.T + b
            if i + 1 < len(layers):
                h = np.maximum(h, 0)
        top2 = np.sort(h, 1)[:, -2:]
        close = (top2[:, 1] - top2[:, 0]) <= MARGIN * np.abs(top2[:, 1])
        near += int(close.sum())
        ok32 = y32[m].reshape(B, -1).argmax(1) == lab
        assert np.all((ok32 == (np.argmax(h, 1) == lab)) | close)
    print(f"{dims} B={B}: {near} of {2 * pairs * B} rows within the margin {MARGIN}")
    pred32 = y32.reshape(2 * pairs, B, -1).argmax(2)
    for mode in ("f16", "f16_any", "bf16", "bf16s"):
        if mode in ("f16", "bf16", "bf16s") and not be.eval_supports_f16(dims, B, act=ACC):
            continue
        if mode == "f16_any" and be.eval_supports_f16(dims, B, act=ACC):
            continue
        kw = _tc_kw(be, mode, theta, table)
        ret, y, _ = _eval(be, dims, theta, table, offs, 0.02, obs, tgt, ACC, B, B * dims[-1], precision=mode, **kw)
        flips = int((y.reshape(2 * pairs, B, -1).argmax(2) != pred32).sum())
        rate = flips / (2 * pairs * B)
        print(f"{mode} {dims} B={B}: {flips} of {2 * pairs * B} predictions differ from fp32 ({rate:.2e}); "
              f"max |return - fp32 return| {np.abs(ret - ret32).max():.4f}")
        assert rate < (2e-3 if mode in ("f16", "f16_any") else 2e-2)


# ------------------------------------------------------------------ goldens, graph replay
def test_goldens_on_the_device(be):
    g = load_golden("es_accuracy_p64.npz")
    dims = [int(d) for d in g["dims"]]
    for gen in range(len(g["returns"])):
        ret, _, _ = _eval(be, dims, g["theta_before"][gen], g["table"], g["offsets"][gen], float(g["sigma"]),
                          g["obs"], g["target"], ACC)
        np.testing.assert_array_equal(ret, g["returns"][gen][:, 0])
    g = load_golden("nsr_accuracy_p32.npz")
    dims = [int(d) for d in g["dims"]]
    for gen in range(len(g["returns"])):
        ret, bcs, _ = _eval(be, dims, g["theta_before"][gen], g["table"], g["offsets"][gen], float(g["sigma"]),
                            g["obs"], g["target"], ACC, int(g["bc_obs"]), int(g["bc_dim"]))
        np.testing.assert_array_equal(ret, g["returns"][gen][:, 0])
        pop, _ = orc.sample_population(g["theta_before"][gen], g["table"], g["offsets"][gen], np.float32(g["sigma"]))
        _, want_bc = ao.evaluate_population(pop, dims, g["obs"], g["target"], int(g["bc_obs"]), int(g["bc_dim"]))
        np.testing.assert_allclose(bcs, want_bc, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("mode,dims,B", [("fp32", [20, 64, 10], 100), ("f16", [64, 128, 256], 256),
                                         ("f16_any", [784, 256, 10], 100)])
def test_graph_replay_equals_eager(be, mode, dims, B):
    pairs = 4
    n, table, theta, obs, _, offs = _tc_problem(dims, B, pairs)
    tgt = _labels_target(np.random.RandomState(2), B, dims[-1])
    kw = _tc_kw(be, mode, theta, table)
    eager, _, _ = _eval(be, dims, theta, table, offs, 0.02, obs, tgt, ACC, precision=mode, **kw)
    ret = be.zeros(2 * pairs)
    args = (dims, dev(be, theta), dev(be, table), dev(be, offs), dev(be, np.arange(pairs, dtype=np.int32)), pairs,
            0.02, dev(be, obs), dev(be, tgt), ret[:pairs], ret[pairs:])
    be.eval_mlp(*args, precision=mode, act=ACC, **kw)          # workspace reserved before the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        be.eval_mlp(*args, precision=mode, act=ACC, **kw)
    ret.zero_()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(ret.cpu().numpy(), eager)


# ------------------------------------------------------------------ learning on minibatches
# settings and bar from the run DESIGN.md §9 reports (one H100, examples/minibatch_classifier.py's dataset)
LEARN = dict(rows=60000, generations=60, population=1024, batch_size=256, seed=0)
LEARN_BAR = 0.4


def test_accuracy_as_the_fitness_learns_the_minibatch_classifier():
    import estorch_b200 as E
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    import minibatch_classifier as mc
    torch.manual_seed(LEARN["seed"])
    x, y = mc.class_conditional(LEARN["rows"], LEARN["seed"])
    es = E.ES(mc.Classifier, E.DeviceAgent, torch.optim.Adam, population_size=LEARN["population"], sigma=0.02,
              agent_kwargs=dict(obs=x, target=y, loss="accuracy", batch_size=LEARN["batch_size"],
                                batch_seed=LEARN["seed"]), optimizer_kwargs={"lr": 0.01})
    assert es._fused and es._sampling and es._act_code() == ACC
    curve = [mc.accuracy(es.policy, x, y)]

    def log():
        if (es.step + 1) % 10 == 0:
            curve.append(mc.accuracy(es.policy, x, y))
    es.log = log
    es.train(n_steps=LEARN["generations"])
    print("full-dataset accuracy every 10 generations:", " ".join(f"{a:.3f}" for a in curve))
    assert curve[-1] > LEARN_BAR > curve[0]
