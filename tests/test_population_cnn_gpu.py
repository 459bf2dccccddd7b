"""Population mode of a generic convolutional policy on the H100: estk_act_cnn (include/estk_act_cnn.h) bit for bit
against the behaviour characteristic of the convolutional evaluate for every code and a range of shapes, each
member's own images against the float64 forward of its materialised fp32 row, isolation between members, repeats
with and without order, sigma = 0, a call whose obs holds more than 2^31 floats, refusals with nothing written,
the reference goldens through ES / NSR-ES on the device, and examples/cnn_catch.py learning."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA GPU", allow_module_level=True)

from estorch_b200 import _capi  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402
from conftest import ROOT  # noqa: E402
from _cnn_oracle import HIDDEN, forward, pack  # noqa: E402
from test_cnn_gpu import _code, _eval, _setup  # noqa: E402
from test_population_cnn_cpu import (check_es_golden, check_nsr_golden, run_es_golden,  # noqa: E402
                                     run_nsr_golden)

TANH = _capi.ESTK_ACT_OUT_TANH
SIGMA = 0.05
BAR = 1e-5
CODES = [h | o for h in HIDDEN for o in (0, TANH)]          # the 10 hidden x output codes of each n_conv
SHAPES = {   # (c, h, w), convs (out_c, k, stride, pad), linears
    "k1_s1": ((3, 5, 5), [(4, 1, 1, 0)], [3]),
    "k8_s4_atari_like": ((2, 36, 36), [(4, 8, 4, 0), (8, 4, 2, 0)], [16, 3]),
    "k5_s2_pad2_three_convs": ((1, 17, 13), [(3, 5, 2, 2), (4, 3, 1, 1), (5, 2, 1, 1)], [6, 5, 4]),
    "k3_s3_pad1_two_linears": ((2, 10, 11), [(3, 3, 3, 1)], [7, 2]),
    "k7_s1_pad0_wide_taps": ((8, 9, 9), [(12, 7, 1, 0)], [300, 5]),
    "slab_64x64": ((1, 64, 64), [(8, 3, 1, 1), (2, 4, 4, 0)], [4]),   # 32,768 activations per image: the slab
}


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _images(shape, B, seed=1):
    return torch.randn(B, *shape, generator=torch.Generator().manual_seed(seed))


def _act(be, dims, code, theta, table, offsets, order, pairs, sigma, obs):
    """estk_act_cnn through the backend: obs [2*pairs, B, ...] (offsets None: [1, B, ...]) -> [M, B, out]."""
    M, B = obs.shape[0], obs.shape[1]
    out = torch.full((M, B, int(dims[-1])), float("nan"), device=be.device)
    be.act_cnn(dims, theta, table, offsets, order, pairs, sigma, obs.contiguous(), out, code)
    torch.cuda.synchronize()
    return out


def _same_images_identity(be, dims, code, B, pairs, seed=0):
    theta, table, offsets, order = _setup(be, dims, code, pairs, seed)
    obs = _images(_shape(dims), B).to(be.device)
    out = int(dims[-1])
    _, bc = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, be.zeros(B, out))
    got = _act(be, dims, code, theta, table, offsets, order, pairs, SIGMA,
               obs.unsqueeze(0).expand(2 * pairs, *obs.shape))
    assert torch.equal(got, bc), (got - bc).abs().max().item()
    # the centre form: theta's outputs, the evaluate's centre BC
    ret, bcc = be.zeros(1), be.zeros(B * out)
    be.eval_cnn_center(dims, theta, obs, be.zeros(B, out), ret, bcc, B, B * out, act=code)
    centre = _act(be, dims, code, theta, None, None, None, 1, 0.0, obs.unsqueeze(0))
    assert torch.equal(centre.reshape(-1), bcc)


def _shape(dims):
    d = int(dims[0]) & 0xffffffff
    return d & 1023, (d >> 10) & 1023, (d >> 20) & 1023


@pytest.mark.parametrize("code", CODES)
@pytest.mark.parametrize("B", [1, 3, 8, 17])
def test_every_code_is_the_evaluate_bc_bit_for_bit(be, code, B):
    shape, convs, linears = SHAPES["k5_s2_pad2_three_convs"]
    dims = pack(shape, convs, linears)
    _same_images_identity(be, dims, _code(len(convs), code), B, 3)


@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("B,pairs", [(1, 1), (3, 64), (8, 3)])
def test_every_shape_is_the_evaluate_bc_bit_for_bit(be, name, B, pairs):
    shape, convs, linears = SHAPES[name]
    _same_images_identity(be, pack(shape, convs, linears), _code(len(convs), 5, TANH), B, pairs)


@pytest.mark.parametrize("B", [1, 4])
def test_a_large_population_is_the_evaluate_bc_bit_for_bit(be, B):
    shape, convs, linears = SHAPES["k3_s3_pad1_two_linears"]
    _same_images_identity(be, pack(shape, convs, linears), _code(len(convs), 1), B, 2048)


def _rows(be, theta, table, offsets, pairs):
    n = theta.numel()
    rows = be.alloc(2 * pairs, n)
    be.perturb_rows(theta, table, offsets, pairs, SIGMA, 0, 2 * pairs, rows)
    torch.cuda.synchronize()
    return rows.cpu().numpy()


def _check_f64(out, rows, dims, code, obs, members):
    for m in members:
        want = forward(rows[m], dims, code, obs[m], dt=np.float64)
        err = np.abs(out[m].astype(np.float64) - want).max() / max(np.abs(want).max(), 1e-30)
        assert err <= BAR, (m, err)


@pytest.mark.parametrize("name", ["k8_s4_atari_like", "k5_s2_pad2_three_convs", "slab_64x64"])
def test_own_images_against_the_float64_forward_and_isolation(be, name):
    shape, convs, linears = SHAPES[name]
    dims, code, pairs, B = pack(shape, convs, linears), _code(len(convs), 4, TANH), 5, 3
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs = torch.randn(2 * pairs, B, *shape, generator=torch.Generator().manual_seed(4)).to(be.device)
    out = _act(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs)
    rows = _rows(be, theta, table, offsets, pairs)
    _check_f64(out.cpu().numpy(), rows, dims, code, obs.cpu().numpy(), range(2 * pairs))
    # changing member m's images changes row m only
    for m in (0, pairs - 1, pairs, 2 * pairs - 1):
        obs2 = obs.clone()
        obs2[m] += 0.5
        out2 = _act(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs2)
        others = [i for i in range(2 * pairs) if i != m]
        assert torch.equal(out2[others], out[others]) and not torch.equal(out2[m], out[m])


def test_the_same_bits_run_to_run_with_and_without_order_and_sigma_zero(be):
    shape, convs, linears = SHAPES["k8_s4_atari_like"]
    dims, code, pairs, B = pack(shape, convs, linears), _code(len(convs), 3), 37, 5
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs = torch.randn(2 * pairs, B, *shape, generator=torch.Generator().manual_seed(6)).to(be.device)
    first = _act(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs)
    perm = torch.randperm(pairs, generator=torch.Generator().manual_seed(2)).to(torch.int32).to(be.device)
    for o in (order, None, perm, order):
        assert torch.equal(_act(be, dims, code, theta, table, offsets, o, pairs, SIGMA, obs), first)
    same = obs[:1].expand(2 * pairs, *obs.shape[1:])
    zero = _act(be, dims, code, theta, table, offsets, order, pairs, 0.0, same)
    centre = _act(be, dims, code, theta, None, None, None, 1, 0.0, obs[:1])
    assert torch.equal(zero, centre.expand_as(zero))


def test_obs_beyond_2_pow_31_floats(be):
    """2 * 2100 * 8 images of 1x256x256 = 2.2e9 floats (8.8 GB): the last members' images lie past 2^31 floats."""
    shape, convs, linears = (1, 256, 256), [(1, 8, 8, 0)], [2]
    dims, code, pairs, B = pack(shape, convs, linears), _code(1, 1), 2100, 8
    assert 2 * pairs * B * 256 * 256 > 2 ** 31
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs = torch.empty(2 * pairs, B, *shape, device=be.device)
    g = torch.Generator(device=be.device).manual_seed(8)
    for m in range(2 * pairs):           # a member's images repeat with period 97 over members, each distinct
        if m < 97:
            obs[m].normal_(generator=g)
        else:
            obs[m].copy_(obs[m % 97]).mul_(1.0 + m / 4096)
    out = _act(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs)
    rows = _rows(be, theta, table, offsets, pairs)
    last = [pairs - 1, 2 * pairs - 2, 2 * pairs - 1]
    _check_f64(out.cpu().numpy(), rows, dims, code, {m: obs[m].cpu().numpy() for m in last}, last)
    del obs


def test_refusals_write_nothing(be):
    shape, convs, linears = (2, 9, 9), [(3, 3, 2, 1)], [4]
    dims, code, pairs, B = pack(shape, convs, linears), _code(1, 0) | _capi.ESTK_ACTIONS, 4, 2
    theta, table, offsets, order = _setup(be, dims, code & ~_capi.ESTK_ACTIONS, pairs)
    obs = torch.randn(2 * pairs, B, *shape).to(be.device)
    out = torch.full((2 * pairs, B, 4), 7.0, device=be.device)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    minus = C.c_void_p(out.data_ptr() + pairs * B * 4 * 4)

    def call(code=code, dd=dims, **over):
        d = _capi.EstkMlpDesc()
        d.n_layers = len(dd) - 1
        for i, w in enumerate(dd):
            d.dims[i] = C.c_int32(int(w)).value
        d.activation = C.c_int32(int(code)).value
        a = dict(ctx=be._ctx, desc=C.byref(d), theta=p(theta), table=p(table), offsets=p(offsets), order=p(order),
                 pairs=pairs, sigma=SIGMA, obs=p(obs), B=B, out_plus=p(out), out_minus=minus, stream=be._stream())
        a.update(over)
        rc = be.lib.estk_act_cnn(*a.values())
        torch.cuda.synchronize()
        return rc
    for over in (dict(theta=None), dict(obs=None), dict(out_plus=None), dict(table=None), dict(out_minus=None),
                 dict(B=0), dict(pairs=0), dict(pairs=(1 << 21) + 1), dict(code=code & ~(3 << 16)),
                 dict(code=code ^ (3 << 16) | _capi.ESTK_LOSS_XENT), dict(code=(code & ~0xff) | _capi.ESTK_CELL_GRU),
                 dict(code=code | 8 << 24), dict(dd=pack(shape, [(3, 3, 2, 3)], linears))):
        assert call(**over) == -1, over
        assert bool((out == 7.0).all())
    assert call() == 0 and not bool((out == 7.0).any())
    # the fixed-batch evaluate still refuses ESTK_ACTIONS with a conv stack
    ret, bc = be.zeros(2 * pairs), be.zeros(2 * pairs, B * 4)
    d = _capi.EstkMlpDesc()
    d.n_layers = len(dims) - 1
    for i, w in enumerate(dims):
        d.dims[i] = C.c_int32(int(w)).value
    d.activation = C.c_int32(int(_capi.ESTK_CNN_N_CONV(1) | _capi.ESTK_ACTIONS)).value
    rc = be.lib.estk_eval_mlp(be._ctx, C.byref(d), _capi.ESTK_PREC_FP32, p(theta), None, p(table), None, p(offsets),
                              p(order), pairs, SIGMA, p(obs), None, B, None, None, p(bc), p(bc), B, B * 4, None,
                              be._stream())
    assert rc == -3


def test_es_population_mode_matches_reference_golden_on_the_device(be):
    check_es_golden(*run_es_golden(be))


def test_nsr_population_mode_matches_reference_golden_on_the_device(be):
    check_nsr_golden(*run_nsr_golden(be))


def test_cnn_catch_example_learns(be):
    spec = importlib.util.spec_from_file_location("cnn_catch", os.path.join(ROOT, "examples", "cnn_catch.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    means, es = ex.train(ex.TEST_GENERATIONS, ex.TEST_POPULATION, backend=be, verbose=False)
    assert es._population and es._is_cnn
    first, last = means[0], float(np.mean(means[-3:]))
    print(f"cnn_catch: generation 0 {first:+.3f}, last three {last:+.3f}")
    assert last - first >= ex.TEST_MARGIN, (first, last)
