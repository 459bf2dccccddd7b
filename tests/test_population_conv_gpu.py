"""Population mode of the conv + VirtualBatchNorm policy on the H100: estk_eval_conv_vbn with
n_actions | ESTK_ACTIONS (estk_act_conv.cu) -- bit-identical to the fp32 evaluate, the stats and act phases
in one call or two, determinism, member isolation, agreement with the numpy forward of materialised rows,
refusals before any launch, ES / NSR-ES in population mode against the reference goldens, and the
pixel-Catch example learning."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA GPU", allow_module_level=True)

from estorch_b200 import _capi  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402
from oracle import es_oracle as orc  # noqa: E402
from _pop_conv_oracle import STATS_FLOATS, AtariPolicy  # noqa: E402
import test_population_conv_cpu as cpu  # noqa: E402

ACTIONS = _capi.ESTK_ACTIONS
f32 = np.float32


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _setup(be, A, pairs, R, seed=0):
    torch.manual_seed(seed)
    g = torch.Generator().manual_seed(seed)
    pol = AtariPolicy(A, torch.zeros(2, 4, 84, 84))
    with torch.no_grad():
        for name, p_ in pol.named_parameters():
            if name.startswith("bn"):
                p_.add_(0.2 * torch.randn(p_.shape, generator=g))
    theta = torch.nn.utils.parameters_to_vector(pol.parameters()).detach().to(be.device).contiguous()
    n = theta.numel()
    table = be.alloc((n + 31) // 32 * 32 + 32 * 4096)
    be.fill_noise_table(table, 11 + seed)
    t16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, t16) == 0
    offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
    be.make_offsets(5 + seed, None, 0, 0, pairs, table.numel(), n, offsets, order)
    xref = torch.rand(R, 4, 84, 84, generator=g).to(be.device)
    return theta, table, t16, offsets, order, xref


def _act(be, A, theta, table, offsets, order, pairs, sigma, xref, obs, table16=None, stats=None, split=False):
    """Both phases (one call, or a stats call then an act call when ``split``); returns (out, stats)."""
    M = 1 if offsets is None else 2 * pairs
    stats = be.alloc(M, STATS_FLOATS) if stats is None else stats
    out = be.alloc(M, obs.shape[1], A)
    t = None if table16 is not None else table
    if split:
        be.act_conv_vbn(A, theta, t, offsets, order, pairs, sigma, xref, None, None, stats, table16=table16)
        be.act_conv_vbn(A, theta, t, offsets, order, pairs, sigma, None, obs, out, stats, table16=table16)
    else:
        be.act_conv_vbn(A, theta, t, offsets, order, pairs, sigma, xref, obs, out, stats, table16=table16)
    return out, stats


def _eval_return(y, t):
    """estk_eval_conv_vbn's fp32 return from the outputs y [B, A] of one member (B*A <= 256, one element per
    thread): d = y - t, d*d per thread, warp_sum_f's xor butterfly over 32 lanes, the 8 warps in order."""
    d = (y - t).astype(f32).reshape(-1)
    v = np.zeros(256, dtype=f32)
    v[:d.size] = d * d
    v = v.reshape(8, 32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[:, lanes ^ o]).astype(f32)
    s = f32(0)
    for w in range(8):
        s = f32(s + v[w, 0])
    return -(s / (f32(y.shape[0]) * f32(y.shape[1])))


CASES = [(2, 1, 1, 1), (5, 3, 4, 3), (128, 32, 8, 64), (2, 32, 4, 3), (5, 1, 8, 64), (128, 3, 1, 1),
         (128, 1, 4, 64), (2, 3, 8, 1), (5, 32, 1, 1)]


@pytest.mark.parametrize("R,B,A,pairs", CASES, ids=lambda v: str(v))
def test_act_outputs_reproduce_the_fp32_evaluate_bit_for_bit(be, R, B, A, pairs):
    sigma = 0.05
    theta, table, t16, offsets, order, xref = _setup(be, A, pairs, R, seed=R + B + A)
    obs = torch.rand(B, 4, 84, 84, device=be.device)
    tgt = torch.randn(B, A, device=be.device)
    scratch = torch.empty(be.conv_scratch_bytes(R, B), dtype=torch.uint8, device=be.device)
    rp, rm = be.zeros(pairs), be.zeros(pairs)
    be.eval_conv_vbn(A, theta, table, offsets, order, pairs, sigma, xref, obs, tgt, rp, rm, scratch)
    out, _ = _act(be, A, theta, table, offsets, order, pairs, sigma, xref,
                  obs[None].expand(2 * pairs, B, 4, 84, 84).contiguous())
    y, t = out.cpu().numpy(), tgt.cpu().numpy()
    want = np.concatenate([rp.cpu().numpy(), rm.cpu().numpy()])
    got = np.array([_eval_return(y[m], t) for m in range(2 * pairs)], dtype=f32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (got[:4], want[:4])
    # the centre: theta's outputs against the centre evaluate
    rc = be.zeros(1)
    be.eval_conv_vbn(A, theta, None, None, None, 1, 0.0, xref, obs, tgt, rc, None, scratch)
    oc, _ = _act(be, A, theta, None, None, None, 1, 0.0, xref, obs[None].contiguous())
    assert _eval_return(oc[0].cpu().numpy(), t).view(np.uint32) == rc.cpu().numpy().view(np.uint32)[0]


def test_split_calls_order_and_either_table_give_the_same_bits(be):
    A, pairs, R, B = 4, 40, 6, 2
    theta, table, t16, offsets, order, xref = _setup(be, A, pairs, R)
    obs = torch.rand(2 * pairs, B, 4, 84, 84, device=be.device)
    ref, ref_stats = _act(be, A, theta, table, offsets, None, pairs, 0.03, xref, obs)
    for o in (None, order):
        for t in (None, t16):
            for split in (False, True):
                out, stats = _act(be, A, theta, table, offsets, o, pairs, 0.03, xref, obs, table16=t, split=split)
                assert torch.equal(out, ref) and torch.equal(stats, ref_stats), (o is None, t is None, split)
    # an act call reuses what an earlier stats call left in the buffer, step after step
    out = be.alloc(2 * pairs, B, A)
    for _ in range(2):
        be.act_conv_vbn(A, theta, table, offsets, order, pairs, 0.03, None, obs, out, ref_stats)
        assert torch.equal(out, ref)


def test_members_are_isolated(be):
    A, pairs, R, B = 4, 16, 4, 3
    theta, table, _, offsets, order, xref = _setup(be, A, pairs, R)
    obs = torch.rand(2 * pairs, B, 4, 84, 84, device=be.device)
    a, _ = _act(be, A, theta, table, offsets, order, pairs, 0.05, xref, obs)
    for m in (0, 5, pairs, 2 * pairs - 1):
        obs2 = obs.clone()
        obs2[m] = torch.rand_like(obs2[m])
        b, _ = _act(be, A, theta, table, offsets, order, pairs, 0.05, xref, obs2)
        changed = (a != b).flatten(1).any(1).nonzero().flatten().tolist()
        assert changed == [m]


def test_act_agrees_with_the_reference_forward_of_materialised_rows(be):
    A, pairs, R, B = 4, 2, 128, 2
    theta, table, _, offsets, _, xref = _setup(be, A, pairs, R)
    obs = torch.rand(2 * pairs, B, 4, 84, 84, device=be.device)
    got, _ = _act(be, A, theta, table, offsets, None, pairs, 0.05, xref, obs)
    rows = be.alloc(2 * pairs, theta.numel())
    be.perturb_rows(theta, table, offsets, pairs, 0.05, 0, 2 * pairs, rows)
    rows, x, xr = rows.cpu().numpy(), obs.cpu().numpy(), xref.cpu().numpy()
    for m in range(2 * pairs):
        want = orc.atari_forward(rows[m], A, xr, x[m])
        err = np.abs(got[m].cpu().numpy() - want).max() / np.abs(want).max()
        assert err < 1e-5, (m, err)


def test_refusals_happen_before_any_launch(be):
    lib = be.lib
    A, pairs, R, B = 4, 3, 4, 2
    theta, table, t16, offsets, order, xref = _setup(be, A, pairs, R)
    obs = torch.rand(2 * pairs, B, 4, 84, 84, device=be.device)
    out = torch.full((2 * pairs, B, A), 7.0, device=be.device)
    stats = torch.full((2 * pairs, STATS_FLOATS), 7.0, device=be.device)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    minus = C.c_void_p(out.data_ptr() + pairs * B * A * 4)

    def call(code, precision=_capi.ESTK_PREC_FP32, x=xref, o=obs, nbytes=stats.numel() * 4):
        return lib.estk_eval_conv_vbn(be._ctx, precision, code, p(theta), p(table), p(t16), p(offsets), p(order),
                                      pairs, 0.05, p(x), R, p(o), None, B, p(out), minus, p(stats), nbytes,
                                      be._stream())
    assert call(A | ACTIONS, _capi.ESTK_PREC_F16) == -3                      # ESTK_ERR_UNSUPPORTED
    for code in (A | ACTIONS | 0x100, A | ACTIONS | 0x8000, ACTIONS, 65 | ACTIONS, A | ACTIONS | (1 << 24)):
        assert call(code) == -1, hex(code)                                   # ESTK_ERR_INVALID
    assert call(A | ACTIONS, nbytes=2 * pairs * STATS_FLOATS * 4 - 4) == -1
    assert call(A | ACTIONS, x=None, o=None) == -1
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()) and bool((stats == 7.0).all())          # nothing was written
    assert call(A | ACTIONS) == 0
    torch.cuda.synchronize()
    assert not bool((out == 7.0).all())


def test_es_population_mode_matches_reference_golden(be):
    cpu.check_es_golden(*cpu.run_es_golden(be))


def test_nsr_population_mode_matches_reference_golden(be):
    cpu.check_nsr_golden(*cpu.run_nsr_golden(be))


def test_pixel_catch_population_learns(be):
    spec = importlib.util.spec_from_file_location("pixel_catch", os.path.join(ROOT, "examples", "pixel_catch.py"))
    pc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(pc)
    means = pc.train(generations=pc.TEST_GENERATIONS, population_size=pc.TEST_POPULATION, seed=0, backend=be,
                     verbose=False)
    print("pixel_catch mean episode reward per generation:", [round(m, 3) for m in means])
    assert np.mean(means[-3:]) > means[0] + pc.TEST_MARGIN, means
