"""Recurrent policies on sequence batches on the H100: the sequence evaluate (estk_eval_mlp with ESTK_CELL_GRU /
ESTK_CELL_LSTM and a return, estk_eval_rnn_seq.cu) bit-identical to T chained ESTK_ACTIONS step launches, its
returns against the fp32 restatement and the float64 forward, determinism, refusals before launch, CUDA-graph
replay, the reference goldens, and a GRU that learns the delayed-recall dataset."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA GPU", allow_module_level=True)

from estorch_b200 import ES, SequenceAgent, _capi  # noqa: E402
from estorch_b200.backend import CudaBackend, mlp_desc  # noqa: E402
from _rnn_oracle import CELL_GRU, CELL_LSTM, param_count, policy_class, state_width  # noqa: E402
from _seq_oracle import (memoryless_best, recall_dataset, seq_forward64, seq_returns32,  # noqa: E402
                         seq_returns64)
from test_population_rnn_cpu import check_es_golden, check_nsr_golden  # noqa: E402
from test_rnn_sequence_cpu import run_es_seq_golden, run_nsr_seq_golden  # noqa: E402

XENT = _capi.ESTK_LOSS_XENT
CODES = [c | rest for c in (CELL_GRU, CELL_LSTM) for rest in (0, 1 << 8, XENT)]
CELL = {CELL_GRU: "gru", CELL_LSTM: "lstm"}
BAR = 2e-6          # max-norm relative distance of outputs and returns from the float64 forward
XENT_ULPS = 8       # cross-entropy returns against the fp32 restatement: CUDA's and numpy's expf / logf differ


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _setup(be, cell, dims, pairs, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    n = param_count(cell, dims)
    theta = ((torch.rand(n, generator=g) * 2 - 1) / np.sqrt(dims[1])).to(be.device)
    table = be.alloc(max(1 << 16, (n + 31) // 32 * 32 + 32 * 4096))
    be.fill_noise_table(table, 11 + seed)
    offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
    be.make_offsets(5 + seed, None, 0, 0, pairs, table.numel(), n, offsets, order)
    return theta, table, offsets, order


def _data(dims, B, T, xent, seed=1):
    g = torch.Generator(device="cpu").manual_seed(seed)
    obs = torch.randn(B, T, dims[0], generator=g)
    if xent:     # class weights, and every third step from t = 2 unscored (an all-zero row)
        tgt = torch.rand(B, T, dims[2], generator=g)
        tgt[:, 2::3] = 0
    else:
        tgt = torch.rand(B, T, dims[2], generator=g) * 1.6 - 0.8
    return obs, tgt


def _seq(be, code, dims, theta, table, offsets, order, pairs, sigma, obs, tgt):
    """The sequence evaluate; returns (returns [2*pairs], y [2*pairs, B, T, out]) read through the BC."""
    B, T = obs.shape[:2]
    per = B * T * dims[2]
    ret, bc = be.alloc(2 * pairs).fill_(float("nan")), be.alloc(2 * pairs, per).fill_(float("nan"))
    be.eval_rnn_seq(dims, theta, table, offsets, order, pairs, sigma, obs, tgt, ret[:pairs], ret[pairs:],
                    bc[:pairs], bc[pairs:], B, per, act=code)
    return ret, bc.view(2 * pairs, B, T, dims[2])


def _chained(be, code, dims, theta, table, offsets, pairs, sigma, obs):
    """T ESTK_ACTIONS step launches, each fed the previous launch's state: y [M, B, T, out]."""
    M = 1 if offsets is None else 2 * pairs
    B, T = obs.shape[:2]
    S = state_width(CELL[code & 0xff], dims[1])
    state = be.zeros(M, B, S)
    ys = []
    for t in range(T):
        x = torch.cat([obs[:, t].expand(M, B, dims[0]), state], -1).contiguous()
        out = be.alloc(M, B, dims[2] + S)
        be.act_rnn(dims, theta, table, offsets, None, pairs, sigma, x, out, code & 0x1ff)
        ys.append(out[..., :dims[2]])
        state = out[..., dims[2]:]
    return torch.stack(ys, 2)


def _rows(be, theta, table, offsets, pairs, sigma):
    rows = be.alloc(2 * pairs, theta.numel())
    be.perturb_rows(theta, table, offsets, pairs, sigma, 0, 2 * pairs, rows)
    return rows.cpu().numpy()


def _maxrel(got, want):
    return float(np.abs(np.asarray(got, np.float64) - want).max() / np.abs(want).max())


# (in, H, out, B, T, pairs): H = 33 and 40 are not multiples of 32; B over {1, 3, 33, 256} (chunks of 1, 4 and
# 16 sequences, a partial last chunk); T over {1, 7, 64}; pairs over {1, 3, 64}.  At H = 256 the activations of
# 16 sequences take most of an SM's shared memory (2*16 rows of 1548 floats for LSTM, 1292 for GRU); at H = 512
# they exceed the budget and stream through the workspace slab.
SHAPES = [(5, 33, 4, 1, 7, 3), (8, 64, 4, 3, 1, 64), (8, 33, 3, 33, 7, 1), (6, 40, 5, 256, 7, 3),
          (8, 64, 4, 3, 64, 3), (8, 256, 4, 20, 7, 3), (8, 512, 4, 6, 3, 2)]


@pytest.mark.parametrize("code", CODES, ids=lambda c: hex(c))
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "-".join(map(str, s)))
def test_outputs_are_t_chained_step_launches_and_returns_the_restatement(be, code, shape):
    i, H, o, B, T, pairs = shape
    dims, cell, sigma, xent = (i, H, o), CELL[code & 0xff], 0.05, bool(code & XENT)
    theta, table, offsets, order = _setup(be, cell, dims, pairs)
    obs, tgt = _data(dims, B, T, xent)
    od, td = obs.to(be.device), tgt.to(be.device)
    ret, y = _seq(be, code, dims, theta, table, offsets, order, pairs, sigma, od, td)
    want_y = _chained(be, code, dims, theta, table, offsets, pairs, sigma, od)
    assert torch.equal(y, want_y)                                        # bit for bit
    yn, rn = y.cpu().numpy(), ret.cpu().numpy()
    r32 = seq_returns32(yn, tgt.numpy(), xent)
    if xent:
        ulp = np.spacing(np.float32(max(1.0, float(np.abs(r32).max()))))
        assert np.abs(rn - r32).max() <= XENT_ULPS * ulp, np.abs(rn - r32).max() / ulp
    else:
        np.testing.assert_array_equal(rn, r32)
    rows = _rows(be, theta, table, offsets, pairs, sigma)
    y64 = seq_forward64(rows, cell, dims, obs.numpy(), bool(code & 0x100))
    r64 = seq_returns64(y64, tgt.numpy(), xent)
    ey, er = _maxrel(yn, y64), _maxrel(rn, r64)
    print(f"{cell} {hex(code)} {shape}: outputs {ey:.2e}, returns {er:.2e} from float64")
    assert ey < BAR and er < BAR, (ey, er)
    # the centre: theta over the same sequences, against one chained member
    rc, bcc = be.zeros(1), be.alloc(B * T * o)
    be.eval_rnn_seq_center(dims, theta, od, td, rc, bcc, B, B * T * o, act=code)
    yc = _chained(be, code, dims, theta, None, None, 1, 0.0, od)
    assert torch.equal(bcc.view(1, B, T, o), yc)
    r32c = seq_returns32(yc.cpu().numpy(), tgt.numpy(), xent)
    assert abs(float(rc[0]) - float(r32c[0])) <= (XENT_ULPS * np.spacing(np.float32(max(1.0, abs(r32c[0]))))
                                                  if xent else 0.0)


def test_same_bits_run_to_run_with_and_without_order_and_sigma_0_gives_the_centre(be):
    for code in CODES:
        cell = CELL[code & 0xff]
        dims, pairs, B, T = (8, 48, 4), 200, 9, 5
        theta, table, offsets, order = _setup(be, cell, dims, pairs)
        obs, tgt = (t.to(be.device) for t in _data(dims, B, T, bool(code & XENT)))
        outs = [_seq(be, code, dims, theta, table, offsets, o, pairs, 0.05, obs, tgt) for o in (None, order)
                for _ in range(2)]
        for r, y in outs[1:]:
            assert torch.equal(r, outs[0][0]) and torch.equal(y, outs[0][1]), hex(code)
        r0, y0 = _seq(be, code, dims, theta, table, offsets, order, pairs, 0.0, obs, tgt)
        rc = be.zeros(1)
        be.eval_rnn_seq_center(dims, theta, obs, tgt, rc, act=code)
        assert torch.equal(r0, rc.expand(2 * pairs)), hex(code)


def test_refusals_happen_before_any_launch(be):
    lib = be.lib
    dims, pairs, B, T = (6, 33, 4), 7, 3, 5
    theta, table, offsets, order = _setup(be, "lstm", dims, pairs)
    obs, tgt = (t.to(be.device) for t in _data(dims, B, T, False))
    ret = be.zeros(2 * pairs)
    per = B * T * dims[2]
    bc = be.zeros(2 * pairs, per)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    minus = lambda t, k: C.c_void_p(t.data_ptr() + pairs * k * 4)  # noqa: E731

    def call(code, precision=_capi.ESTK_PREC_FP32, steps=T, tg=p(tgt), rp=p(ret), centre_out=None, dd=dims):
        d = mlp_desc(dd, code, steps=steps) if len(dd) == 3 else mlp_desc(dd, code)
        return lib.estk_eval_mlp(be._ctx, C.byref(d), precision, p(theta), None, p(table), None, p(offsets),
                                 p(order), pairs, 0.05, p(obs), tg, B, rp, minus(ret, 1), p(bc), minus(bc, per), B,
                                 per, centre_out, be._stream())
    for code in CODES:
        for prec in (_capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S, _capi.ESTK_PREC_F16_ANY):
            assert call(code, prec) == -3                                      # ESTK_ERR_UNSUPPORTED
        assert call(code, centre_out=p(ret)) == -3
        assert call(code, steps=0) == -1                                       # T < 1
        assert call(code, tg=None) == -1
        assert call(code, rp=None) == -1
        assert call(code, dd=(6, 33, 33, 4)) == -1                             # n_layers must be 2
    for code in (CELL_GRU | XENT | 0x100, CELL_LSTM | XENT | 0x100):           # XENT with a Tanh output
        assert call(code) == -1
    torch.cuda.synchronize()
    assert float(ret.abs().sum()) == 0.0 and float(bc.abs().sum()) == 0.0    # nothing was written
    assert call(CELL_LSTM) == 0


def test_graph_replay_equals_eager(be):
    code, dims, pairs, B, T = CELL_GRU | 0x100, (8, 64, 4), 64, 16, 12
    theta, table, offsets, order = _setup(be, "gru", dims, pairs)
    obs, tgt = (t.to(be.device) for t in _data(dims, B, T, False))
    eager = _seq(be, code, dims, theta, table, offsets, order, pairs, 0.05, obs, tgt)
    ret, bc = be.zeros(2 * pairs), be.zeros(2 * pairs, B * T * 4)
    side = torch.cuda.Stream(be.device)
    side.wait_stream(torch.cuda.current_stream(be.device))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        graph.capture_begin()
        be.eval_rnn_seq(dims, theta, table, offsets, order, pairs, 0.05, obs, tgt, ret[:pairs], ret[pairs:],
                        bc[:pairs], bc[pairs:], B, B * T * 4, act=code)
        graph.capture_end()
    torch.cuda.current_stream(be.device).wait_stream(side)
    for _ in range(2):
        ret.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(ret, eager[0]) and torch.equal(bc.view_as(eager[1]), eager[1])


def test_es_gru_sequence_matches_reference_golden(be):
    check_es_golden(*run_es_seq_golden(be))


def test_nsr_lstm_cross_entropy_sequence_matches_reference_golden(be):
    check_nsr_golden(*run_nsr_seq_golden(be))


RECALL_BAR = -0.01     # an H100 measured -0.0079 at generation 28 and -0.0000 from generation 40 (DESIGN §9)


def test_gru_learns_the_delayed_recall_dataset(be):
    """Seed 0, P = 256: the centre's return passes RECALL_BAR within 60 generations; no memoryless policy can do
    better than memoryless_best() (-0.183)."""
    assert RECALL_BAR > memoryless_best()
    obs, tgt = recall_dataset(copies=4)
    torch.manual_seed(0)
    rewards = []
    es = ES(policy_class("gru", False), SequenceAgent, torch.optim.Adam, population_size=256, sigma=0.05,
            policy_kwargs={"dims": (4, 32, 3)}, agent_kwargs=dict(obs=obs, target=tgt, loss="cross_entropy"),
            optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 18, _backend=be)
    es.log = lambda: rewards.append(float(es.episode_reward))
    assert es._fused and es._is_rnn and not es._population
    es.train(n_steps=60)
    print("delayed recall, centre return per generation:", [round(r, 4) for r in rewards])
    assert max(rewards) > RECALL_BAR, rewards
