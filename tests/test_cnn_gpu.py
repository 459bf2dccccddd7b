"""Convolutional policies on fixed batches on the H100: the CNN evaluate (estk_eval_mlp with n_conv in bits 24-31,
estk_eval_cnn.cu) against the float64 forward of every member's fp32 weights, bit-exact cross-checks (materialised
rows, the fp32 MLP evaluate, sigma = 0, repeats with and without order), refusals before any launch, CUDA-graph
replay, and ES training a small CNN in fused mode."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA GPU", allow_module_level=True)

from estorch_b200 import ES, DeviceAgent, _capi  # noqa: E402
from estorch_b200.backend import CudaBackend, cnn_desc  # noqa: E402
from _cnn_oracle import HIDDEN, image_task, layer_shapes, pack, param_count, policy_class, unpack  # noqa: E402
from test_cnn_cpu import run_es_cnn_golden, run_nsr_cnn_golden  # noqa: E402
from test_population_rnn_cpu import check_es_golden, check_nsr_golden  # noqa: E402

XENT, TANH = _capi.ESTK_LOSS_XENT, _capi.ESTK_ACT_OUT_TANH
BAR = 1e-5          # max-norm relative distance of returns and outputs from the float64 forward
SIGMA = 0.05


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _code(n_conv, hidden=0, rest=0):
    return hidden | rest | n_conv << 24


def _setup(be, dims, code, pairs, seed=0):
    n_conv = code >> 24
    torch.manual_seed(seed)
    pol = policy_class(n_conv, HIDDEN[code & 0xff], bool(code & TANH))(dims)
    theta = torch.nn.utils.parameters_to_vector(pol.parameters()).detach().to(be.device).contiguous()
    n = theta.numel()
    assert n == param_count(dims, n_conv)
    table = be.alloc(max(1 << 16, (n + 31) // 32 * 32 + 32 * 4096))
    be.fill_noise_table(table, 11 + seed)
    offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
    be.make_offsets(5 + seed, None, 0, 0, pairs, table.numel(), n, offsets, order)
    return theta, table, offsets, order


def _data(shape, B, out, xent, seed=1):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(B, *shape, generator=g)
    tgt = torch.rand(B, out, generator=g) if xent else torch.rand(B, out, generator=g) * 1.6 - 0.8
    return obs, tgt


def _eval(be, dims, code, theta, table, offsets, order, pairs, sigma, obs, tgt):
    """Returns [2*pairs] and every member's outputs [2*pairs, B, out] (read through the BC)."""
    B, out = tgt.shape
    ret, bc = be.zeros(2 * pairs), be.zeros(2 * pairs, B * out)
    be.eval_cnn(dims, theta, table, offsets, order, pairs, sigma, obs, tgt, ret[:pairs], ret[pairs:], bc[:pairs],
                bc[pairs:], B, B * out, act=code)
    torch.cuda.synchronize()
    return ret, bc.view(2 * pairs, B, out)


def _forward64(rows, dims, code, obs, chunk=128):
    """The float64 forward of fp32 rows [M, n] on obs [B, c, h, w]: grouped convolutions, members as groups."""
    n_conv = code >> 24
    shape, convs, linears = unpack(dims, n_conv)
    shapes, _ = layer_shapes(shape, convs, linears)
    act = {"relu": torch.relu, "tanh": torch.tanh, "elu": F.elu, "silu": F.silu,
           "leaky_relu": F.leaky_relu}[HIDDEN[code & 0xff]]
    outs = []
    for m0 in range(0, rows.shape[0], chunk):
        R = rows[m0: m0 + chunk].double()
        M, B = R.shape[0], obs.shape[0]
        h = obs.double().unsqueeze(0).expand(M, *obs.shape).permute(1, 0, 2, 3, 4).reshape(B, M * shape[0],
                                                                                             *shape[1:])
        i = 0
        for li, (ws, bl) in enumerate(shapes):
            sz = int(np.prod(ws))
            w, b = R[:, i: i + sz].reshape(M, *ws), R[:, i + sz: i + sz + bl]
            i += sz + bl
            if li < n_conv:
                _, _, s, p = convs[li]
                h = act(F.conv2d(h, w.reshape(M * ws[0], *ws[1:]), b.reshape(-1), stride=s, padding=p, groups=M))
                if li == n_conv - 1:
                    h = h.reshape(B, M, -1).permute(1, 0, 2)          # [M, B, C*H*W] in (c, h, w) order
            else:
                h = torch.einsum("mbk,mok->mbo", h, w) + b[:, None]
                if li + 1 < len(shapes):
                    h = act(h)
        outs.append(torch.tanh(h) if code & TANH else h)
    return torch.cat(outs)


def _returns64(y, tgt, xent):
    t = tgt.double()[None]
    if xent:
        return (t * torch.log_softmax(y, -1)).sum(-1).mean(1)
    return -((y - t) ** 2).mean((1, 2))


def _rel(got, want):
    return float((got.double() - want).abs().max() / want.abs().max())


# (input shape, convs (out_c, k, stride, pad), linear widths, B, pairs)
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
CODES = [(h, rest) for h in HIDDEN for rest in (0, TANH, XENT)]
WORST = {}


def _check(be, name, hidden, rest):
    shape, convs, linears, B, pairs = CASES[name]
    dims, code = pack(shape, convs, linears), _code(len(convs), hidden, rest)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, linears[-1], bool(rest & XENT)))
    ret, y = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    rows = be.alloc(2 * pairs, theta.numel())
    be.perturb_rows(theta, table, offsets, pairs, SIGMA, 0, 2 * pairs, rows)
    y64 = _forward64(rows, dims, code, obs)
    r64 = _returns64(y64, tgt, bool(rest & XENT))
    ey, er = _rel(y, y64), _rel(ret, r64)
    WORST[(name, hidden, rest)] = (ey, er)
    print(f"{name} code={code:#x}: outputs {ey:.2e}, returns {er:.2e}")
    assert ey < BAR and er < BAR


@pytest.mark.parametrize("hidden,rest", CODES)
def test_every_code_against_float64(be, hidden, rest):
    _check(be, "c3_k3_p1", hidden, rest)


@pytest.mark.parametrize("name", [n for n in CASES if n != "c3_k3_p1"])
def test_shapes_against_float64(be, name):
    i = list(CASES).index(name)
    hidden, rest = CODES[(3 * i + 1) % len(CODES)]
    _check(be, name, hidden, rest)
    if name == "mnist":
        _check(be, name, 0, XENT)


def test_a_member_is_its_materialised_row(be):
    shape, convs, linears, B, pairs = CASES["atari_small"]
    dims, code = pack(shape, convs, linears), _code(2, 4, 0)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, linears[-1], False))
    ret, y = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    rows = be.alloc(2 * pairs, theta.numel())
    be.perturb_rows(theta, table, offsets, pairs, SIGMA, 0, 2 * pairs, rows)
    for m in (0, 5, pairs, 2 * pairs - 1):
        one, bc = be.zeros(1), be.zeros(B * linears[-1])
        be.eval_cnn_center(dims, rows[m].contiguous(), obs, tgt, one, bc, B, B * linears[-1], act=code)
        torch.cuda.synchronize()
        assert torch.equal(one[0], ret[m]) and torch.equal(bc.view(B, -1), y[m]), m


@pytest.mark.parametrize("rest", [0, TANH])
def test_a_full_kernel_conv_is_the_mlp_first_linear(be, rest):
    """k = h = w, stride 1, pad 0: the conv is the fp32 MLP evaluate's first Linear on the flattened image."""
    shape, convs, linears, B, pairs = (3, 5, 5), [(8, 5, 1, 0)], [6, 4], 37, 16
    dims, code = pack(shape, convs, linears), _code(1, 1, rest)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, 4, False))
    _, y = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    ret, bc = be.zeros(2 * pairs), be.zeros(2 * pairs, B * 4)
    be.eval_mlp([75, 8, 6, 4], theta, table, offsets, order, pairs, SIGMA, obs.reshape(B, -1).contiguous(), tgt,
                ret[:pairs], ret[pairs:], bc[:pairs], bc[pairs:], B, B * 4, act=1 | rest)
    torch.cuda.synchronize()
    assert torch.equal(bc.view_as(y), y)


def test_sigma_zero_and_repeats(be):
    shape, convs, linears, B, pairs = CASES["four_convs"]
    dims, code = pack(shape, convs, linears), _code(4, 3, XENT)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, linears[-1], True))
    r0, y0 = _eval(be, dims, code, theta, table, offsets, order, pairs, 0.0, obs, tgt)
    one, bc = be.zeros(1), be.zeros(B * linears[-1])
    be.eval_cnn_center(dims, theta, obs, tgt, one, bc, B, B * linears[-1], act=code)
    torch.cuda.synchronize()
    assert torch.equal(r0, one.expand_as(r0)) and torch.equal(y0, bc.view(1, B, -1).expand_as(y0))
    runs = [_eval(be, dims, code, theta, table, offsets, o, pairs, SIGMA, obs, tgt) for o in (None, order, order)]
    for r, y in runs[1:]:
        assert torch.equal(r, runs[0][0]) and torch.equal(y, runs[0][1])


def test_a_large_image_runs_on_a_bounded_slab():
    """3x512x512 with 16 channels: 67 MB of activations per CTA.  The slab grid is capped by the workspace budget
    (1 GB), not by the resident CTAs (which would need tens of GB); the results are those of the float64 forward."""
    be2 = CudaBackend()
    shape, convs, linears, B, pairs = (3, 512, 512), [(16, 3, 1, 1), (4, 16, 16, 0)], [4], 2, 2
    dims, code = pack(shape, convs, linears), _code(2, 0, 0)
    theta, table, offsets, order = _setup(be2, dims, code, pairs)
    obs, tgt = (t.to(be2.device) for t in _data(shape, B, 4, False))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(be2.device)[0]
    ret, y = _eval(be2, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    grown = free0 - torch.cuda.mem_get_info(be2.device)[0]
    assert grown < (4 << 30), grown          # the 1 GB slab plus slack: every resident CTA's slab would be ~27 GB
    rows = be2.alloc(2 * pairs, theta.numel())
    be2.perturb_rows(theta, table, offsets, pairs, SIGMA, 0, 2 * pairs, rows)
    y64 = _forward64(rows, dims, code, obs)
    assert _rel(y, y64) < BAR and _rel(ret, _returns64(y64, tgt, False)) < BAR


def test_refusals_happen_before_any_launch(be):
    lib = be.lib
    shape, convs, linears, B, pairs = (3, 9, 9), [(4, 3, 2, 1)], [5], 3, 4
    dims, code = pack(shape, convs, linears), _code(1)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, 5, False))
    ret, bc = be.zeros(2 * pairs), be.zeros(2 * pairs, B * 5)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    minus = lambda t, k: C.c_void_p(t.data_ptr() + pairs * k * 4)  # noqa: E731

    def call(code, precision=_capi.ESTK_PREC_FP32, dd=dims, tg=p(tgt), centre_out=None):
        d = _capi.EstkMlpDesc()
        d.n_layers = len(dd) - 1
        for i, w in enumerate(dd):
            d.dims[i] = C.c_int32(int(w)).value
        d.activation = C.c_int32(int(code)).value
        return lib.estk_eval_mlp(be._ctx, C.byref(d), precision, p(theta), None, p(table), None, p(offsets),
                                 p(order), pairs, SIGMA, p(obs), tg, B, p(ret), minus(ret, 1), p(bc),
                                 minus(bc, B * 5), B, B * 5, centre_out, be._stream())
    for c in (code, _code(1, 1, TANH), _code(1, 0, XENT)):
        for prec in (_capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S, _capi.ESTK_PREC_F16_ANY):
            assert call(c, prec) == -3                                          # ESTK_ERR_UNSUPPORTED
            assert call(c, prec, dd=(0, 0)) == -3                               # before the packed fields
        assert call(c, centre_out=p(ret)) == -3
    assert call(1 << 24, _capi.ESTK_PREC_F16_ANY, dd=(0, 0)) == -3
    for c in (_code(1, 0, _capi.ESTK_ACTIONS), _code(1, _capi.ESTK_CELL_GRU), _code(1, _capi.ESTK_CELL_LSTM, TANH)):
        assert call(c) == -3
    for c in (-1, 8 << 24, 2 | 1 << 24, _code(1, 0, XENT | TANH), _code(1, 0, 0x20000), _code(2)):
        assert call(c) == -1, hex(c)                                            # ESTK_ERR_INVALID
    bad_dims = [pack((0, 9, 9), convs, linears), pack(shape, [(0, 3, 2, 1)], linears),
                pack(shape, [(4, 3, 2, 3)], linears), pack(shape, [(4, 12, 1, 1)], linears),
                pack(shape, [(4, 3, 0, 1)], linears), pack(shape, convs, [0]), pack(shape, convs, [])]
    for dd in bad_dims:
        assert call(code, dd=dd) == -1, dd
    assert call(code, tg=None) == -1
    assert call(code, precision=9) == -1
    torch.cuda.synchronize()
    assert float(ret.abs().sum()) == 0.0 and float(bc.abs().sum()) == 0.0    # nothing was written
    assert call(code) == 0
    for prec in range(5):
        assert lib.estk_eval_mlp_supported(C.byref(cnn_desc(dims, code)), prec, B) == 0


def test_graph_replay_equals_eager(be):
    shape, convs, linears, B, pairs = CASES["mnist"]
    dims, code = pack(shape, convs, linears), _code(2, 0, XENT)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, 10, True))
    eager = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    ret, bc = be.zeros(2 * pairs), be.zeros(2 * pairs, B * 10)
    side = torch.cuda.Stream(be.device)
    side.wait_stream(torch.cuda.current_stream(be.device))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        graph.capture_begin()
        be.eval_cnn(dims, theta, table, offsets, order, pairs, SIGMA, obs, tgt, ret[:pairs], ret[pairs:],
                    bc[:pairs], bc[pairs:], B, B * 10, act=code)
        graph.capture_end()
    torch.cuda.current_stream(be.device).wait_stream(side)
    for _ in range(2):
        ret.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(ret, eager[0]) and torch.equal(bc.view_as(eager[1]), eager[1])


def test_es_cnn_matches_reference_golden(be):
    check_es_golden(*run_es_cnn_golden(be))


def test_nsr_cnn_cross_entropy_matches_reference_golden(be):
    check_nsr_golden(*run_nsr_cnn_golden(be))


def test_es_trains_a_cnn_classifier_in_fused_mode(be):
    obs, tgt = image_task(256, seed=3)
    dims = pack((1, 12, 12), [(8, 3, 2, 1), (8, 3, 2, 1)], [4])
    torch.manual_seed(0)
    rewards = []
    es = ES(policy_class(2, "relu", False), DeviceAgent, torch.optim.Adam, population_size=256, sigma=0.05,
            policy_kwargs={"dims": dims}, agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy"),
            optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 18, _backend=be)
    es.log = lambda: rewards.append(float(es.episode_reward))
    assert es._fused and es._is_cnn and not es._population and es._precision == "fp32"
    es.train(n_steps=30)
    print("cnn classifier, centre return per generation:", [round(r, 4) for r in rewards])
    assert rewards[-1] > rewards[0] + 0.5


def test_example_cnn_classifier_learns():
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "cnn_classifier.py")
    spec = importlib.util.spec_from_file_location("cnn_classifier", path)
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    first, last, acc0, acc1 = ex.main(generations=ex.TEST_GENERATIONS, population=ex.TEST_POPULATION)
    print(f"cnn_classifier: accuracy {acc0:.3f} -> {acc1:.3f}")
    assert acc1 >= acc0 + ex.TEST_MARGIN
