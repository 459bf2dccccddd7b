"""Recurrent policies in population mode on the H100: estk_eval_mlp with ESTK_CELL_GRU / ESTK_CELL_LSTM and
ESTK_ACTIONS (estk_act_rnn.cu) against the float64 forward of every member's fp32 weights, a 100-step closed
loop against the numpy fp32 restatement, determinism, member isolation, refusals before launch, ES / NSR-ES
against the reference goldens, and a GRU population that learns the recall task."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA GPU", allow_module_level=True)

from estorch_b200 import ES, _capi  # noqa: E402
from estorch_b200.backend import CudaBackend, mlp_desc  # noqa: E402
import test_population_rnn_cpu as cpu  # noqa: E402
from _rnn_oracle import (CELL_GRU, CELL_LSTM, RecallAgent, forward64, param_count, policy_class,  # noqa: E402
                         state_width, step32)

CODES = [c | o for c in (CELL_GRU, CELL_LSTM) for o in (0, 1 << 8)]
CELL = {CELL_GRU: "gru", CELL_LSTM: "lstm"}
BAR = 2e-6        # max-norm relative distance of one step from the float64 forward (an H100 measured <= 3.8e-7)


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _setup(be, cell, dims, pairs, seed=0):
    """theta at torch's initialisation scale (U(-1/sqrt(H), 1/sqrt(H))), the noise table and its exact fp16 copy,
    and the offsets / order of ``pairs`` pairs."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    n = param_count(cell, dims)
    theta = ((torch.rand(n, generator=g) * 2 - 1) / np.sqrt(dims[1])).to(be.device)
    table = be.alloc(max(1 << 16, (n + 31) // 32 * 32 + 32 * 4096))
    be.fill_noise_table(table, 11 + seed)
    t16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, t16) == 0
    offsets, order = be.zeros(max(pairs, 1), dtype=torch.int64), be.zeros(max(pairs, 1), dtype=torch.int32)
    be.make_offsets(5 + seed, None, 0, 0, max(pairs, 1), table.numel(), n, offsets, order)
    return theta, table, t16, offsets, order


def _inputs(cell, dims, M, B, seed=1):
    """[M, B, in + S]: observations N(0, 1), h in (-1, 1), c N(0, 1)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    i, H, _ = dims
    parts = [torch.randn(M, B, i, generator=g), torch.rand(M, B, H, generator=g) * 2 - 1]
    if cell == "lstm":
        parts.append(torch.randn(M, B, H, generator=g))
    return torch.cat(parts, -1)


def _step(be, code, dims, theta, table, offsets, pairs, sigma, xs, order=None, table16=None):
    cell = CELL[code & 0xff]
    out = be.alloc(xs.shape[0], xs.shape[1], dims[2] + state_width(cell, dims[1]))
    out.fill_(float("nan"))
    be.act_rnn(dims, theta, None if table16 is not None else table, offsets, order, pairs, sigma, xs, out, code,
               table16=table16)
    return out


def _rows(be, theta, table, offsets, pairs, sigma):
    rows = be.alloc(2 * pairs, theta.numel())
    be.perturb_rows(theta, table, offsets, pairs, sigma, 0, 2 * pairs, rows)
    return rows.cpu().numpy()


def _maxrel(got, want):
    return float(np.abs(np.asarray(got, np.float64) - want).max() / np.abs(want).max())


# (in, H, out, B, pairs): H not a multiple of 32, B over {1, 3, 8, 9}, pairs over {1, 3, 64, 2048}; at B = 8 and
# H = 256 the activations (2*8 rows of 1560 floats) do not fit the shared-memory budget and stream through the slab
SHAPES = [(24, 40, 4, 1, 3), (24, 33, 4, 3, 64), (5, 70, 2, 9, 1), (24, 256, 4, 8, 3), (24, 24, 4, 1, 2048)]


@pytest.mark.parametrize("code", CODES, ids=lambda c: hex(c))
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "-".join(map(str, s)))
def test_every_code_matches_the_float64_forward(be, code, shape):
    i, H, o, B, pairs = shape
    dims, cell, sigma = (i, H, o), CELL[code & 0xff], 0.05
    theta, table, t16, offsets, order = _setup(be, cell, dims, pairs)
    xs = _inputs(cell, dims, 2 * pairs, B)
    got = _step(be, code, dims, theta, table, offsets, pairs, sigma, xs.to(be.device).contiguous(), order=order)
    want = forward64(_rows(be, theta, table, offsets, pairs, sigma), cell, dims, xs.numpy(), bool(code & 0x100))
    err = _maxrel(got.cpu().numpy(), want)
    print(f"{cell} {hex(code)} {shape}: max-norm relative {err:.2e}")
    assert err < BAR, err
    # the centre: theta's step
    xc = _inputs(cell, dims, 1, B, seed=2)
    gc = _step(be, code, dims, theta, None, None, 1, 0.0, xc.to(be.device).contiguous())
    wc = forward64(theta.cpu().numpy()[None], cell, dims, xc.numpy(), bool(code & 0x100))
    assert _maxrel(gc.cpu().numpy(), wc) < BAR


CLOSED_LOOP_BAR = 4e-6    # 100 steps of the state fed back: the kernel against the numpy fp32 restatement
                          # (an H100 measured at most 3.1e-7)


@pytest.mark.parametrize("code", CODES, ids=lambda c: hex(c))
def test_a_100_step_closed_loop_stays_near_the_fp32_restatement(be, code):
    dims, pairs, B, sigma = (6, 48, 3), 8, 2, 0.05
    cell = CELL[code & 0xff]
    S = state_width(cell, dims[1])
    theta, table, _, offsets, order = _setup(be, cell, dims, pairs, seed=3)
    rows = _rows(be, theta, table, offsets, pairs, sigma)
    g = torch.Generator(device="cpu").manual_seed(4)
    xs = torch.randn(100, 2 * pairs, B, dims[0], generator=g)
    sd = torch.zeros(2 * pairs, B, S, device=be.device)
    sn = np.zeros((2 * pairs, B, S), np.float32)
    worst = 0.0
    for t in range(100):
        out = _step(be, code, dims, theta, table, offsets, pairs, sigma,
                    torch.cat([xs[t].to(be.device), sd], -1).contiguous(), order=order)
        ref = step32(rows, cell, dims, np.concatenate([xs[t].numpy(), sn], -1), bool(code & 0x100))
        worst = max(worst, _maxrel(out.cpu().numpy(), ref))
        sd, sn = out[..., dims[2]:].contiguous(), ref[..., dims[2]:]
    print(f"{cell} {hex(code)}: 100-step closed loop, worst max-norm relative {worst:.2e}")
    assert worst < CLOSED_LOOP_BAR, worst


def test_same_bits_run_to_run_with_and_without_order_from_either_table(be):
    for code in CODES:
        cell = CELL[code & 0xff]
        dims, pairs, B = (24, 64, 4), 300, 2
        theta, table, t16, offsets, order = _setup(be, cell, dims, pairs)
        xs = _inputs(cell, dims, 2 * pairs, B).to(be.device).contiguous()
        outs = [_step(be, code, dims, theta, table, offsets, pairs, 0.05, xs, order=o, table16=t)
                for o in (None, order) for t in (None, t16) for _ in range(2)]
        for o in outs[1:]:
            assert torch.equal(o, outs[0]), hex(code)


def test_members_are_isolated(be):
    for code in (CELL_GRU, CELL_LSTM | 0x100):
        cell = CELL[code & 0xff]
        dims, pairs, B = (17, 33, 5), 64, 3
        theta, table, _, offsets, order = _setup(be, cell, dims, pairs)
        xs = _inputs(cell, dims, 2 * pairs, B).to(be.device)
        a = _step(be, code, dims, theta, table, offsets, pairs, 0.05, xs.contiguous(), order=order)
        keep = torch.tensor([0, 5, pairs, pairs + 63], device=be.device)
        xs2 = torch.randn_like(xs) * 3       # other members' observations and states change
        xs2[keep] = xs[keep]
        b = _step(be, code, dims, theta, table, offsets, pairs, 0.05, xs2.contiguous(), order=order)
        assert torch.equal(a[keep], b[keep])
        assert not torch.equal(a, b)


def test_refusals_happen_before_any_launch(be):
    lib = be.lib
    dims, pairs, B = (17, 33, 5), 7, 3
    theta, table, t16, offsets, order = _setup(be, "lstm", dims, pairs)
    xs = _inputs("lstm", dims, 2 * pairs, B).to(be.device).contiguous()
    per = B * (dims[2] + 2 * dims[1])
    out = be.zeros(2 * pairs, B, dims[2] + 2 * dims[1])
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    minus = C.c_void_p(out.data_ptr() + pairs * per * 4)

    def call(code, precision, bc_plus, dd=dims):
        d = mlp_desc(dd, code)
        return lib.estk_eval_mlp(be._ctx, C.byref(d), precision, p(theta), p(theta), p(table), p(t16), p(offsets),
                                 p(order), pairs, 0.05, p(xs), None, B, None, None, bc_plus, minus, B, per, None,
                                 be._stream())
    act = _capi.ESTK_ACTIONS
    for prec in (_capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S, _capi.ESTK_PREC_F16_ANY):
        for code in CODES:
            assert call(code | act, prec, p(out)) == -3                          # ESTK_ERR_UNSUPPORTED
        assert call(CELL_LSTM | act, prec, p(out), (17, 33, 33, 5)) == -3
    for code in (CELL_LSTM, CELL_LSTM | 0x100, CELL_LSTM | _capi.ESTK_LOSS_XENT, CELL_GRU | 0x20000,
                 CELL_GRU | 0x30200, CELL_LSTM | 0x70000, 10 | act, 7 | act):
        assert call(code, _capi.ESTK_PREC_FP32, p(out)) == -1, hex(code)         # ESTK_ERR_INVALID
    assert call(CELL_LSTM | act, _capi.ESTK_PREC_FP32, p(out), (17, 33)) == -1    # n_layers must be 2
    assert call(CELL_LSTM | act, _capi.ESTK_PREC_FP32, p(out), (17, 33, 33, 5)) == -1
    assert call(CELL_LSTM | act, _capi.ESTK_PREC_FP32, None) == -1
    torch.cuda.synchronize()
    assert float(out.abs().sum()) == 0.0                                          # nothing was written
    assert call(CELL_LSTM | act, _capi.ESTK_PREC_FP32, p(out)) == 0


def test_es_gru_population_mode_matches_reference_golden(be):
    cpu.check_es_golden(*cpu.run_es_golden(be))


def test_nsr_lstm_population_mode_matches_reference_golden(be):
    cpu.check_nsr_golden(*cpu.run_nsr_golden(be))


def test_gru_population_learns_the_recall_task(be):
    """Seed 0, P = 128: the centre policy's return passes -0.2 within 60 generations; no memoryless policy can
    do better than RecallAgent.MEMORYLESS_BEST (-0.569)."""
    torch.manual_seed(0)
    rewards = []
    es = ES(policy_class("gru", True), RecallAgent, torch.optim.Adam, population_size=128, sigma=0.05,
            policy_kwargs={"dims": (4, 32, 3)}, optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 16,
            _backend=be)
    es.log = lambda: rewards.append(float(es.episode_reward))
    assert es._population and es._is_rnn
    es.train(n_steps=60)
    print("recall task, centre return per generation:", [round(r, 3) for r in rewards])
    assert rewards[0] < RecallAgent.MEMORYLESS_BEST + 0.05
    assert max(rewards) > -0.2, rewards
