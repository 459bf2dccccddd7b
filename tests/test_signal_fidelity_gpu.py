"""Evaluate kernels against a float64 evaluate on what ES consumes of their returns: the antithetic
differences D_j = R+_j - R-_j, the centred ranks and the gradient (tests/_fp64_signal.py), across sigma,
the weight scale and the observation scale.

fp32 back ends: every member's rank is its float64 rank, except where a float64 neighbour lies within the
fp32 error bound tau of the two returns; every return lies within its tau; where the ranks agree with those
of the float64 returns (rounded to fp32), the device's gradient is the same bits.

Tensor-core modes: the kernel adds no error beyond its rounding model (its signal metrics stay within a
small factor of the CPU emulation's), and inside the domain ES documents for it the gradient is within
3e-2 (rel-L2) of the float64-return gradient.  Cells outside the domain are reported, not asserted.  One
JSON line per cell, prefixed SIGNAL_FIDELITY."""
import json

import numpy as np
import pytest
import torch

from estorch_b200 import _capi
from estorch_b200.backend import CudaBackend
from estorch_b200.estorch import AUTO_F16_MIN_SIGMA
from oracle import es_oracle as orc
import _mlp_oracle as mlp
import _fp64_signal as sig
from _oracle_backend import OracleBackend

pytestmark = pytest.mark.gpu

PAIRS = 32
GRAD_BAR = 3e-2


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _dev(be, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(be.device)


def _linear_theta(dims, scale, seed=0):
    torch.manual_seed(seed)
    mods = [torch.nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])]
    flat = torch.cat([t.detach().reshape(-1) for m in mods for t in (m.weight, m.bias)]).numpy()
    return (flat * np.float32(scale)).astype(np.float32)


def _noise(be, n, pairs, seed=7):
    table = be.alloc(max(1 << 16, (n + 31) // 32 * 32 + 32 * 16 * pairs))
    be.fill_noise_table(table, seed)
    offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(seed + 1, None, 0, 0, pairs, table.numel(), n, offs, order)
    return table, offs, order


def _report(**cell):
    print("SIGNAL_FIDELITY " + json.dumps(cell, sort_keys=True))


def _fp32_bar(be, what, ret, r64, tau, table, offs, order, theta_d, **cell):
    r = ret.cpu().numpy()
    ranks, g = sig.device_gradient(be, ret, table, offs, order, theta_d)
    ranks64, g64 = sig.device_gradient(be, _dev(be, r64.astype(np.float32)), table, offs, order, theta_d)
    m = sig.signal_metrics(r, r64, g, g64)
    viol, pinned = sig.rank_violations(r, r64, tau)
    m.update(pinned=pinned, err_over_tau=float(np.max(np.abs(r - r64) / tau)), rank_violations=int(viol.size))
    _report(backend=what, **cell, **m)
    assert np.all(np.abs(r - r64) <= tau), (what, cell, m)
    assert viol.size == 0, (what, cell, viol, m)
    if np.array_equal(ranks, ranks64):
        np.testing.assert_array_equal(g, g64)
    if cell["sigma"] == 0.02:       # the bar binds: members with no float64 neighbour within the bound exist
        assert pinned > 0, (what, cell, m)


# ------------------------------------------------------------------ fp32 back ends
FP32_SIGMAS, FP32_SCALES = (0.02, 1e-3, 2e-4), (1.0, 8.0)


@pytest.mark.parametrize("sigma", FP32_SIGMAS)
@pytest.mark.parametrize("scale", FP32_SCALES)
@pytest.mark.parametrize("B", [1, 256])
@pytest.mark.parametrize("shape", ["dense", "wide"])
def test_fp32_mlp_keeps_float64_ranks(be, shape, B, scale, sigma):
    """The dense shared-memory kernel ([16, 64, 64, 4]) and the streamed wide kernel ([1088, 64, 8])."""
    dims = [16, 64, 64, 4] if shape == "dense" else [1088, 64, 8]
    theta = _linear_theta(dims, scale)
    table, offs, order = _noise(be, theta.size, PAIRS)
    g = np.random.RandomState(1)
    obs, tgt = g.standard_normal((B, dims[0])).astype(np.float32), g.standard_normal((B, dims[-1])).astype(np.float32)
    th_d = _dev(be, theta)
    ret = be.zeros(2 * PAIRS)
    be.eval_mlp(dims, th_d, table, offs, order, PAIRS, sigma, _dev(be, obs), _dev(be, tgt), ret[:PAIRS], ret[PAIRS:])
    rows = sig.members(theta, table.cpu().numpy(), offs.cpu().numpy(), sigma)
    r64, tau = sig.mlp_reference(rows, dims, obs, tgt)
    _fp32_bar(be, f"fp32 {shape} {dims}", ret, r64, tau, table, offs, order, th_d, B=B, scale=scale, sigma=sigma)


@pytest.mark.parametrize("sigma", FP32_SIGMAS)
@pytest.mark.parametrize("scale", FP32_SCALES)
@pytest.mark.parametrize("B", [1, 64])
def test_fp32_gru_sequence_keeps_float64_ranks(be, B, scale, sigma):
    import _rnn_oracle as rnn
    dims, T = (5, 32, 3), 6
    g = np.random.RandomState(3)
    theta = ((g.rand(rnn.param_count("gru", dims)) * 2 - 1) / np.sqrt(dims[1]) * scale).astype(np.float32)
    table, offs, order = _noise(be, theta.size, PAIRS)
    obs = g.standard_normal((B, T, dims[0])).astype(np.float32)
    tgt = (g.rand(B, T, dims[2]) * 1.6 - 0.8).astype(np.float32)
    th_d = _dev(be, theta)
    ret = be.zeros(2 * PAIRS)
    be.eval_rnn_seq(dims, th_d, table, offs, order, PAIRS, sigma, _dev(be, obs), _dev(be, tgt), ret[:PAIRS],
                    ret[PAIRS:], act=_capi.ESTK_CELL_GRU)
    rows = sig.members(theta, table.cpu().numpy(), offs.cpu().numpy(), sigma)
    r64, tau = sig.seq_reference(rows, "gru", list(dims), obs, tgt)
    _fp32_bar(be, "fp32 gru sequence", ret, r64, tau, table, offs, order, th_d, B=B, scale=scale, sigma=sigma)


@pytest.mark.parametrize("sigma", FP32_SIGMAS)
@pytest.mark.parametrize("scale", FP32_SCALES)
@pytest.mark.parametrize("B", [1, 64])
def test_fp32_cnn_keeps_float64_ranks(be, B, scale, sigma):
    import _cnn_oracle as cnn
    dims, code = cnn.pack((3, 12, 12), [(8, 3, 2, 1), (16, 3, 1, 0)], [16, 4]), 2 << 24
    torch.manual_seed(0)
    pol = cnn.policy_class(2)(dims)
    theta = (torch.nn.utils.parameters_to_vector(pol.parameters()).detach().numpy() * scale).astype(np.float32)
    table, offs, order = _noise(be, theta.size, PAIRS)
    g = np.random.RandomState(4)
    obs, tgt = g.standard_normal((B, 3, 12, 12)).astype(np.float32), g.standard_normal((B, 4)).astype(np.float32)
    th_d = _dev(be, theta)
    ret = be.zeros(2 * PAIRS)
    be.eval_cnn(dims, th_d, table, offs, order, PAIRS, sigma, _dev(be, obs), _dev(be, tgt), ret[:PAIRS], ret[PAIRS:],
                act=code)
    rows = sig.members(theta, table.cpu().numpy(), offs.cpu().numpy(), sigma)
    r64, tau = sig.cnn_reference(rows, dims, code, obs, tgt)
    _fp32_bar(be, "fp32 cnn", ret, r64, tau, table, offs, order, th_d, B=B, scale=scale, sigma=sigma)


def _atari(be, scale, pairs, B, R=16):
    import _vbn_frames as vf
    theta = vf.policy_row(4, "init", 0).astype(np.float32) * np.float32(scale)
    xref, obs = vf.frames("unit", R, B, seed=2)
    tgt = np.random.RandomState(5).standard_normal((B, 4)).astype(np.float32)
    table, offs, order = _noise(be, theta.size, pairs)
    return theta.astype(np.float32), xref, obs, tgt, table, offs, order


def _conv(be, mode, theta_d, table, offs, order, pairs, sigma, xref, obs, tgt):
    tb16 = None
    if mode == "f16":
        tb16 = be.alloc(table.numel(), dtype=torch.float16)
        assert be.shadow_f16(table, tb16) == 0
    scratch = torch.empty(be.conv_scratch_bytes(xref.shape[0], obs.shape[0], mode), dtype=torch.uint8,
                          device=be.device)
    ret = be.zeros(2 * pairs)
    be.eval_conv_vbn(4, theta_d, table, offs, order, pairs, sigma, _dev(be, xref), _dev(be, obs), _dev(be, tgt),
                     ret[:pairs], ret[pairs:], scratch, precision=mode, table16=tb16)
    return ret


@pytest.mark.parametrize("sigma", FP32_SIGMAS)
@pytest.mark.parametrize("scale", FP32_SCALES)
@pytest.mark.parametrize("B", [1, 8])
def test_fp32_conv_vbn_keeps_float64_ranks(be, B, scale, sigma):
    pairs = 8
    theta, xref, obs, tgt, table, offs, order = _atari(be, scale, pairs, B)
    th_d = _dev(be, theta)
    ret = _conv(be, "fp32", th_d, table, offs, order, pairs, sigma, xref, obs, tgt)
    rows = sig.members(theta, table.cpu().numpy(), offs.cpu().numpy(), sigma)
    r64, tau = sig.conv_vbn_reference(rows, 4, xref, obs, tgt)
    _fp32_bar(be, "fp32 conv_vbn", ret, r64, tau, table, offs, order, th_d, B=B, scale=scale, sigma=sigma)


# ------------------------------------------------------------------ tensor-core modes
def in_domain(mode, sigma, scale, obs_scale):
    """The documented accuracy domain: f16 / f16_any at sigma >= AUTO_F16_MIN_SIGMA (where "auto" picks f16)
    with weights up to 8x init, observations of any scale; bf16 / bf16s at sigma >= 0.05 up to 8x init."""
    if mode in ("f16", "f16_any"):
        return sigma >= AUTO_F16_MIN_SIGMA and scale <= 8
    return sigma >= 0.05 and scale <= 8


# (mode, dims, hidden, loss): the cluster kernel, the streamed kernel and a 784-wide cross-entropy head
CONFIGS = {
    "f16_relu": ("f16", [64, 256, 256, 32], "relu", "mse"),
    "f16_tanh": ("f16", [64, 256, 256, 32], "tanh", "mse"),
    "f16_silu": ("f16", [64, 256, 256, 32], "silu", "mse"),
    "f16_any_relu": ("f16_any", [33, 200, 70, 10], "relu", "mse"),
    "f16_any_silu_xent": ("f16_any", [784, 256, 10], "silu", "xent"),
    "f16_any_tanh_xent": ("f16_any", [784, 256, 10], "tanh", "xent"),
    "bf16_relu": ("bf16", [64, 256, 256, 32], "relu", "mse"),
    "bf16s_relu": ("bf16s", [64, 256, 256, 32], "relu", "mse"),
}
SIGMAS = (0.05, 0.02, 5e-3, 1e-3, 2e-4)
# a covering set: the default path on the whole sigma x scale grid and both off-unit observation scales;
# every other configuration on sigma x {1, 8} and one off-unit observation scale
CELLS = ([("f16_relu", s, w, 1.0) for s in SIGMAS for w in (1.0, 4.0, 8.0)] +
         [("f16_relu", s, w, o) for s, w in ((0.02, 1.0), (1e-3, 4.0), (5e-3, 8.0)) for o in (1e-3, 100.0)] +
         [(c, s, w, 1.0) for c in CONFIGS if c != "f16_relu" for s in SIGMAS for w in (1.0, 8.0)] +
         [(c, 5e-3, 4.0, o) for c in CONFIGS if c != "f16_relu" for o in (1e-3, 100.0)])


def _tc_call(be, mode, dims, th_d, table, offs, order, sigma, obs_d, tgt_d, act):
    extra = {}
    if mode in ("f16", "f16_any"):
        extra["table16"] = be.alloc(table.numel(), dtype=torch.float16)
        assert be.shadow_f16(table, extra["table16"]) == 0
    elif mode == "bf16s":
        extra["table16"] = be.alloc(table.numel(), dtype=torch.bfloat16)
        extra["theta16"] = be.alloc(th_d.numel(), dtype=torch.bfloat16)
        be.shadow_bf16(table, extra["table16"])
        be.shadow_bf16(th_d, extra["theta16"])
    ret = be.zeros(2 * PAIRS)
    be.eval_mlp(dims, th_d, table, offs, order, PAIRS, sigma, obs_d, tgt_d, ret[:PAIRS], ret[PAIRS:], precision=mode,
                act=act, **extra)
    return ret


@pytest.mark.parametrize("config,sigma,scale,obs_scale", CELLS)
def test_tensor_core_signal_vs_rounding_model_and_domain(be, config, sigma, scale, obs_scale):
    mode, dims, hidden, loss = CONFIGS[config]
    B = 256
    theta = _linear_theta(dims, scale)
    table, offs, order = _noise(be, theta.size, PAIRS)
    g = np.random.RandomState(1)
    obs = (g.standard_normal((B, dims[0])) * obs_scale).astype(np.float32)
    tgt = (np.eye(dims[-1], dtype=np.float32)[g.randint(0, dims[-1], B)] if loss == "xent" else
           g.standard_normal((B, dims[-1])).astype(np.float32))
    th_d = _dev(be, theta)
    ret = _tc_call(be, mode, dims, th_d, table, offs, order, sigma, _dev(be, obs), _dev(be, tgt),
                   mlp.code(hidden, "identity", loss))
    table_h, offs_h = table.cpu().numpy(), offs.cpu().numpy()
    rows = sig.members(theta, table_h, offs_h, sigma)
    r64, _ = sig.mlp_reference(rows, dims, obs, tgt, hidden, "identity", loss)
    model_rows = rows
    if mode == "bf16s":
        model_rows = OracleBackend._exact_biases(orc.sample_population_bf16s(theta, table_h, offs_h, sigma), rows,
                                                 dims)
    r_model, _ = mlp.evaluate_population(model_rows, dims, obs, tgt, mlp.code(hidden, "identity", loss), mode)
    _, g64 = sig.device_gradient(be, _dev(be, r64.astype(np.float32)), table, offs, order, th_d)
    _, g = sig.device_gradient(be, ret, table, offs, order, th_d)
    _, g_model = sig.device_gradient(be, _dev(be, r_model), table, offs, order, th_d)
    r = ret.cpu().numpy()
    m = sig.signal_metrics(r, r64, g, g64)
    mm = sig.signal_metrics(r_model, r64, g_model, g64)
    pairs = PAIRS
    d64 = r64[:pairs] - r64[pairs:]
    kernel_vs_model = float(np.max(np.abs((r[:pairs] - r[pairs:]) - (r_model[:pairs] - r_model[pairs:])))
                            / d64.std())
    domain = in_domain(mode, sigma, scale, obs_scale)
    _report(config=config, mode=mode, dims=dims, hidden=hidden, loss=loss, sigma=sigma, scale=scale,
            obs_scale=obs_scale, in_domain=domain, kernel=m, model=mm, diff_kernel_vs_model_over_std=kernel_vs_model)
    # the kernel adds no error beyond its rounding model
    assert kernel_vs_model < 0.1, kernel_vs_model
    assert m["returns_max_rel"] <= 2 * mm["returns_max_rel"] + 1e-6
    assert m["diff_wrong_sign"] <= 2 * mm["diff_wrong_sign"] + 2 / pairs
    assert m["grad_rel_l2"] <= 2 * mm["grad_rel_l2"] + 1.5e-2
    if domain:
        assert m["grad_rel_l2"] <= GRAD_BAR, m


@pytest.mark.parametrize("sigma,scale", [(0.02, 1.0), (5e-3, 8.0), (1e-3, 1.0), (1e-3, 8.0)])
def test_conv_f16_signal_vs_fp32_kernel(be, sigma, scale):
    """The conv + VirtualBatchNorm "f16" kernel (hi + lo fp16 operands, 22 bits): its rounding model is the
    fp32 kernel's, so its signal metrics stay within a small factor of the fp32 kernel's."""
    pairs, B = 16, 8
    theta, xref, obs, tgt, table, offs, order = _atari(be, scale, pairs, B)
    th_d = _dev(be, theta)
    r16 = _conv(be, "f16", th_d, table, offs, order, pairs, sigma, xref, obs, tgt)
    r32 = _conv(be, "fp32", th_d, table, offs, order, pairs, sigma, xref, obs, tgt)
    rows = sig.members(theta, table.cpu().numpy(), offs.cpu().numpy(), sigma)
    r64, _ = sig.conv_vbn_reference(rows, 4, xref, obs, tgt)
    _, g64 = sig.device_gradient(be, _dev(be, r64.astype(np.float32)), table, offs, order, th_d)
    m16 = sig.signal_metrics(r16.cpu().numpy(), r64, sig.device_gradient(be, r16, table, offs, order, th_d)[1], g64)
    m32 = sig.signal_metrics(r32.cpu().numpy(), r64, sig.device_gradient(be, r32, table, offs, order, th_d)[1], g64)
    _report(config="conv_vbn_f16", sigma=sigma, scale=scale, kernel=m16, fp32_kernel=m32)
    assert m16["returns_max_rel"] <= 8 * m32["returns_max_rel"] + 1e-6
    assert m16["diff_wrong_sign"] <= 2 * m32["diff_wrong_sign"] + 2 / pairs
    assert m16["grad_rel_l2"] <= 2 * m32["grad_rel_l2"] + GRAD_BAR
