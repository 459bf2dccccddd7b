"""Every reader of the noise table on a table of 2^31 + 2^22 entries: rows past element 2^31 (fp16 byte 2^32) and
past fp32 byte 2^32.

The table is real: 8 GiB of fp32 unit normals and their exact 4 GiB fp16 copy, allocated whole, so a row address
that a kernel truncates to 32 bits still lands inside the allocation and shows up as wrong values, not as a fault.

Bars:
  relocation identity -- the rows of the big table named by the big offsets, copied into a small table at small
      offsets, give the SAME BITS through every entry point that reads ``table`` or ``table16`` (no kernel's
      arithmetic depends on the offset value, and the same ``order`` array is passed to both runs);
  gradient -- both rank + gradient entry points within 1e-5 (max-norm relative) of a float64 gather-matmul of the
      rows the offsets name, ranks bit-exact, theta / m / v the oracle's Adam step;
  offsets -- estk_make_offsets bit-exact against the oracle up to ESTK_MAX_TABLE_LEN, on both sort paths.

Offsets are chosen by hand so that the boundaries are hit by construction: 0, a row across element 2^30 (fp32
byte 2^32), a row across element 2^31, exactly 2^31, rows between 2^31 and the end, and the last slot.  Larger
populations fill their other pairs from estk_make_offsets: half over the whole table and half over the rows past
2^31 (a uniform draw over the whole table puts only 0.2 % of its rows there).
"""
import os

import numpy as np
import pytest
import torch

from estorch_b200 import _capi
from oracle import es_oracle as orc
from conftest import rel_err

pytestmark = pytest.mark.gpu

TABLE_LEN = (1 << 31) + (1 << 22)
E30, E31 = 1 << 30, 1 << 31
GIB = 1 << 30
# the fp32 table, its fp16 copy and headroom for the small tables, populations and the float64 reference
NEED_BYTES = 6 * TABLE_LEN + 2 * GIB
SIGMA = 0.02


def _skip_without_memory(need):
    free, _total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / GIB:.1f} GiB of free device memory for a {TABLE_LEN}-entry noise table and its "
                    f"fp16 copy; {free / GIB:.1f} GiB free")


class Big:
    """The module's table: ``t`` fp32 [TABLE_LEN], ``t16`` its exact fp16 copy."""

    def __init__(self, be):
        self.be = be
        self.t = be.alloc(TABLE_LEN)
        be.fill_noise_table(self.t, 0x5EED)
        self.t16 = be.alloc(TABLE_LEN, dtype=torch.float16)
        assert be.shadow_f16(self.t, self.t16) == 0


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


@pytest.fixture(scope="module")
def big(be):
    _skip_without_memory(NEED_BYTES)
    torch.cuda.reset_peak_memory_stats(be.device)
    b = Big(be)
    yield b
    print(f"peak device memory {torch.cuda.max_memory_allocated(be.device) / GIB:.2f} GiB")
    del b
    torch.cuda.empty_cache()


def ceil32(n):
    return (n + 31) // 32 * 32


def fixed_offsets(n):
    """Hand-chosen rows of an n-parameter policy, every one a multiple of 32 and inside the table."""
    n_pad = ceil32(n)
    back = 32 * max(1, n_pad // 64)              # a row starting here runs across the boundary
    assert n > back
    last = TABLE_LEN - n_pad
    return [0, E30 - back, E31 - back, E31, E31 + 32, (E31 + last) // 2 // 32 * 32, last - 4096, last]


def offsets_of(be, n, pairs, seed=7):
    """int64 device offsets [pairs]: the fixed rows, then estk_make_offsets draws (half over the whole table,
    half over the rows past 2^31); and int32 ``order``, the stable argsort of the offsets."""
    fixed = fixed_offsets(n)[:pairs]
    offs = torch.tensor(fixed, dtype=torch.int64, device=be.device)
    rest = pairs - len(fixed)
    if rest > 0:
        whole, upper = be.alloc(rest - rest // 2, dtype=torch.int64), be.alloc(rest // 2, dtype=torch.int64)
        be.make_offsets(seed, None, 0, 0, whole.numel(), TABLE_LEN, n, whole)
        if upper.numel():
            be.make_offsets(seed + 1, None, 0, 0, upper.numel(), TABLE_LEN - E31, n, upper)
        drawn = torch.cat([whole, upper + E31])
        if rest >= 2:
            assert int((drawn >= E31).sum()) * 4 >= rest
        if whole.numel() >= 64:
            assert int((whole >= E30).sum()) * 4 >= whole.numel()      # past fp32 byte 2^32
        offs = torch.cat([offs, drawn])
    o = offs.cpu().numpy()
    assert (o % 32 == 0).all() and (o >= 0).all() and (o + ceil32(n) <= TABLE_LEN).all()
    assert (o >= E31).sum() >= min(pairs, 4)
    order = torch.from_numpy(np.argsort(o, kind="stable").astype(np.int32)).to(be.device)
    return offs.contiguous(), order


def relocate(big, offs, n, f16=True, bf16=False):
    """The rows the big offsets name, copied into a small table at j * n_pad: (table, table16 | None,
    bf16 table | None, small offsets)."""
    be, n_pad, pairs = big.be, ceil32(n), offs.numel()
    small = be.alloc(pairs * n_pad)
    idx = torch.arange(n_pad, device=be.device)
    rows = small.view(pairs, n_pad)
    for j0 in range(0, pairs, 8):
        rows[j0:j0 + 8] = big.t[offs[j0:j0 + 8, None] + idx[None, :]]
    s16 = sb16 = None
    if f16:
        s16 = be.alloc(small.numel(), dtype=torch.float16)
        assert be.shadow_f16(small, s16) == 0
    if bf16:
        sb16 = be.alloc(small.numel(), dtype=torch.bfloat16)
        be.shadow_bf16(small, sb16)
    soffs = torch.arange(pairs, dtype=torch.int64, device=be.device) * n_pad
    return small, s16, sb16, soffs


def same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    assert a.shape == b.shape and a.dtype == b.dtype
    assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                       b.view(torch.int32) if b.dtype == torch.float32 else b), \
        f"{int((a != b).sum())} of {a.numel()} entries differ"


def mlp_theta(be, dims, seed=3):
    g = torch.Generator().manual_seed(seed)
    parts = []
    for i in range(len(dims) - 1):
        bound = 1.0 / dims[i] ** 0.5
        parts.append((torch.rand(dims[i] * dims[i + 1] + dims[i + 1], generator=g) * 2 - 1) * bound)
    return torch.cat(parts).to(be.device)


def randn(be, *shape, seed=1, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(be.device)


# ------------------------------------------------------------------ rows
def test_perturb_rows_relocated_and_exact(be, big):
    n, pairs = 4610, 8
    offs, _ = offsets_of(be, n, pairs)
    theta = randn(be, n, scale=0.1)
    small, _, _, soffs = relocate(big, offs, n, f16=False)
    out = {}
    for name, t, o in (("big", big.t, offs), ("small", small, soffs)):
        rows, eps = be.alloc(2 * pairs, n), be.alloc(2 * pairs, n)
        be.perturb_rows(theta, t, o, pairs, SIGMA, 0, 2 * pairs, rows, eps)
        out[name] = (rows, eps)
    same_bits(out["big"][0], out["small"][0])
    same_bits(out["big"][1], out["small"][1])
    # and each row is theta +- fp32(sigma * T[off:off+n]) of the row the offset names
    t = big.t[offs[:, None] + torch.arange(n, device=be.device)[None, :]]
    e = torch.tensor(SIGMA, dtype=torch.float32, device=be.device) * t
    same_bits(out["big"][1], torch.cat([e, -e]))
    same_bits(out["big"][0], torch.cat([theta + e, theta - e]))


# ------------------------------------------------------------------ MLP evaluate and population mode
# (dims, B): the cluster kernel's shapes for fp32 / f16 / bf16 / bf16s; a shape it refuses for f16_any
MLP_CASES = {"fp32": ([64, 128, 32], 256), "f16": ([64, 128, 32], 256), "bf16": ([64, 128, 32], 256),
             "bf16s": ([64, 128, 32], 256), "f16_any": ([4, 64, 64, 2], 100)}


@pytest.mark.parametrize("precision", list(MLP_CASES))
def test_eval_mlp_relocated(be, big, precision):
    dims, B = MLP_CASES[precision]
    if precision == "f16_any":
        assert not be.eval_supports_f16(dims, B) and be.eval_supports_f16_any(dims, B)
    elif precision != "fp32":
        assert be.eval_supports_f16(dims, B) and be.eval_supports_bf16(dims, B)
    n, pairs = orc.mlp_param_count(dims), 64
    offs, order = offsets_of(be, n, pairs)
    theta = mlp_theta(be, dims)
    obs, tgt = randn(be, B, dims[0], seed=4), randn(be, B, dims[-1], seed=5)
    bf16s = precision == "bf16s"
    small, s16, sb16, soffs = relocate(big, offs, n, f16=not bf16s, bf16=bf16s)
    th16 = tb16 = None
    if bf16s:
        th16 = be.alloc(n, dtype=torch.bfloat16)
        be.shadow_bf16(theta, th16)
        tb16 = be.alloc(TABLE_LEN, dtype=torch.bfloat16)     # the big table's bf16 shadow: this case only
        be.shadow_bf16(big.t, tb16)
    runs = {"big": (big.t, tb16 if bf16s else big.t16, offs), "small": (small, sb16 if bf16s else s16, soffs)}
    out = {}
    for name, (t, t16, o) in runs.items():
        ret = torch.full((2 * pairs,), float("nan"), device=be.device)
        be.eval_mlp(dims, theta, t, o, order, pairs, SIGMA, obs, tgt, ret[:pairs], ret[pairs:], precision=precision,
                    theta16=th16, table16=None if precision in ("fp32", "bf16") else t16)
        out[name] = ret
    assert torch.isfinite(out["big"]).all()
    same_bits(out["big"], out["small"])


@pytest.mark.parametrize("form", ["table", "table16"])
def test_act_mlp_relocated(be, big, form):
    dims, B, pairs = [4, 64, 64, 2], 3, 64
    n = orc.mlp_param_count(dims)
    offs, order = offsets_of(be, n, pairs)
    theta = mlp_theta(be, dims)
    obs = randn(be, 2 * pairs, B, dims[0], seed=6)
    small, s16, _, soffs = relocate(big, offs, n)
    out = {}
    for name, t, t16, o in (("big", big.t, big.t16, offs), ("small", small, s16, soffs)):
        y = torch.full((2 * pairs, B, dims[-1]), float("nan"), device=be.device)
        be.act_mlp(dims, theta, t, o, order, pairs, SIGMA, obs, y, table16=t16 if form == "table16" else None)
        out[name] = y
    assert torch.isfinite(out["big"]).all()
    same_bits(out["big"], out["small"])


# ------------------------------------------------------------------ convolutional policies
CNN_SHAPE = ((2, 36, 36), [(4, 8, 4, 0), (8, 4, 2, 0)], [16, 3])     # the Atari-like shape of the CNN tests


def _cnn():
    from _cnn_oracle import pack, param_count
    shape, convs, linears = CNN_SHAPE
    dims = pack(shape, convs, linears)
    code = len(convs) << _capi.ESTK_CNN_SHIFT       # ReLU hidden, identity output, squared error
    return dims, code, param_count(dims, len(convs))


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_eval_cnn_relocated(be, big, precision):
    dims, code, n = _cnn()
    B, pairs = 5, 16
    if precision == "tf32":
        assert be.eval_supports_tf32_cnn(dims, B, code)
    offs, order = offsets_of(be, n, pairs)
    theta = randn(be, n, seed=8, scale=0.1)
    obs, tgt = randn(be, B, *CNN_SHAPE[0], seed=9), randn(be, B, CNN_SHAPE[2][-1], seed=10)
    small, _, _, soffs = relocate(big, offs, n, f16=False)
    out = {}
    for name, t, o in (("big", big.t, offs), ("small", small, soffs)):
        ret = torch.full((2 * pairs,), float("nan"), device=be.device)
        be.eval_cnn(dims, theta, t, o, order, pairs, SIGMA, obs, tgt, ret[:pairs], ret[pairs:], precision=precision,
                    act=code)
        out[name] = ret
    assert torch.isfinite(out["big"]).all()
    same_bits(out["big"], out["small"])


def test_act_cnn_relocated(be, big):
    dims, code, n = _cnn()
    B, pairs = 2, 16
    offs, order = offsets_of(be, n, pairs)
    theta = randn(be, n, seed=8, scale=0.1)
    obs = randn(be, 2 * pairs, B, *CNN_SHAPE[0], seed=11)
    small, _, _, soffs = relocate(big, offs, n, f16=False)
    out = {}
    for name, t, o in (("big", big.t, offs), ("small", small, soffs)):
        y = torch.full((2 * pairs, B, CNN_SHAPE[2][-1]), float("nan"), device=be.device)
        be.act_cnn(dims, theta, t, o, order, pairs, SIGMA, obs, y, code)
        out[name] = y
    assert torch.isfinite(out["big"]).all()
    same_bits(out["big"], out["small"])


# ------------------------------------------------------------------ conv + VirtualBatchNorm policy
def _atari(be, A):
    n = sum(int(np.prod(s)) for _, s in orc.atari_param_layout(A))
    theta = randn(be, n, seed=12, scale=0.02)
    layout, k = orc.atari_param_layout(A), 0
    for name, s in layout:                           # VBN scales near 1, as a trained policy has them
        size = int(np.prod(s))
        if name in ("bn1.w", "bn2.w"):
            theta[k:k + size] += 1.0
        k += size
    g = torch.Generator().manual_seed(13)
    xref = (torch.rand(2, 4, 84, 84, generator=g) * 255).to(be.device)
    return n, theta, xref


@pytest.mark.parametrize("precision", ["fp32", "f16"])
def test_eval_conv_vbn_relocated(be, big, precision):
    A, B, pairs = 4, 2, 8
    n, theta, xref = _atari(be, A)
    offs, order = offsets_of(be, n, pairs)
    obs = (torch.rand(B, 4, 84, 84, generator=torch.Generator().manual_seed(14)) * 255).to(be.device)
    tgt = randn(be, B, A, seed=15)
    small, s16, _, soffs = relocate(big, offs, n)
    scratch = torch.empty(be.conv_scratch_bytes(2, B, precision), dtype=torch.uint8, device=be.device)
    out = {}
    for name, t, t16, o in (("big", big.t, big.t16, offs), ("small", small, s16, soffs)):
        rp, rm = torch.full((pairs,), float("nan"), device=be.device), torch.full((pairs,), float("nan"),
                                                                                device=be.device)
        be.eval_conv_vbn(A, theta, t, o, order, pairs, SIGMA, xref, obs, tgt, rp, rm, scratch, precision=precision,
                         table16=t16 if precision == "f16" else None)
        out[name] = torch.cat([rp, rm])
    assert torch.isfinite(out["big"]).all()
    same_bits(out["big"], out["small"])


@pytest.mark.parametrize("form", ["table", "table16"])
def test_act_conv_vbn_relocated(be, big, form):
    A, B, pairs = 4, 1, 8
    n, theta, xref = _atari(be, A)
    offs, order = offsets_of(be, n, pairs)
    obs = (torch.rand(2 * pairs, B, 4, 84, 84, generator=torch.Generator().manual_seed(16)) * 255).to(be.device)
    small, s16, _, soffs = relocate(big, offs, n)
    out = {}
    for name, t, t16, o in (("big", big.t, big.t16, offs), ("small", small, s16, soffs)):
        stats = be.alloc(2 * pairs, _capi.ESTK_CONV_VBN_STATS_FLOATS)
        y = torch.full((2 * pairs, B, A), float("nan"), device=be.device)
        be.act_conv_vbn(A, theta, t, o, order, pairs, SIGMA, xref, obs, y, stats,
                        table16=t16 if form == "table16" else None)
        out[name] = (y, stats)
    assert torch.isfinite(out["big"][0]).all()
    same_bits(out["big"][0], out["small"][0])
    same_bits(out["big"][1], out["small"][1])


# ------------------------------------------------------------------ recurrent policies
@pytest.mark.parametrize("form", ["table", "table16"])
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_act_rnn_relocated(be, big, cell, form):
    from _rnn_oracle import CELLS, param_count, state_width
    dims, B, pairs = (5, 32, 3), 2, 16
    n, S = param_count(cell, dims), state_width(cell, dims[1])
    offs, order = offsets_of(be, n, pairs)
    theta = randn(be, n, seed=17, scale=0.2)
    obs = randn(be, 2 * pairs, B, dims[0] + S, seed=18)
    small, s16, _, soffs = relocate(big, offs, n)
    out = {}
    for name, t, t16, o in (("big", big.t, big.t16, offs), ("small", small, s16, soffs)):
        y = torch.full((2 * pairs, B, dims[-1] + S), float("nan"), device=be.device)
        be.act_rnn(dims, theta, t, o, order, pairs, SIGMA, obs, y, CELLS[cell],
                   table16=t16 if form == "table16" else None)
        out[name] = y
    assert torch.isfinite(out["big"]).all()
    same_bits(out["big"], out["small"])


@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_eval_rnn_seq_relocated(be, big, cell):
    from _rnn_oracle import CELLS, param_count
    dims, B, T, pairs = (5, 32, 3), 4, 6, 16
    n = param_count(cell, dims)
    offs, order = offsets_of(be, n, pairs)
    theta = randn(be, n, seed=19, scale=0.2)
    obs, tgt = randn(be, B, T, dims[0], seed=20), randn(be, B, T, dims[-1], seed=21)
    small, _, _, soffs = relocate(big, offs, n, f16=False)
    out = {}
    for name, t, o in (("big", big.t, offs), ("small", small, soffs)):
        ret = torch.full((2 * pairs,), float("nan"), device=be.device)
        be.eval_rnn_seq(dims, theta, t, o, order, pairs, SIGMA, obs, tgt, ret[:pairs], ret[pairs:], act=CELLS[cell])
        out[name] = ret
    assert torch.isfinite(out["big"]).all()
    same_bits(out["big"], out["small"])


# ------------------------------------------------------------------ rank + gradient
# n = 4610: n % 8 == 2, the 256-thread pair-split path (PS > 1); n = 1,001,760: the 512-thread column-split path
GRAD_N = [4610, 1001760]


def _rank_grad(be, fn, returns, table, offs, order, n, theta=None, m=None, v=None, world=1, key=None):
    """One rank + gradient call: fn "adam" (estk_rank_grad_adam) -> (ranks, grad, theta, m, v);
    fn "raw" (estk_rank_grad, world shards, rank-major returns when world > 1) -> (ranks, grad_sum) per shard.
    A shard's reduction order is the stable argsort of ``key[shard]`` (default: its offsets), so that a relocated
    run can keep the big table's order."""
    from estorch_b200.backend import adam_desc, new_state
    P = returns.numel()
    if fn == "adam":
        th, mm, vv, g = theta.clone(), m.clone(), v.clone(), be.zeros(n)
        ranks = be.zeros(P, dtype=torch.int32)
        be.rank_grad_adam(returns, None, 1.0, 0.0, P, table, offs, order, th, mm, vv, new_state(be.device),
                          adam_desc(lr=0.01), ranks, None, g)
        return ranks, g, th, mm, vv
    pairs, pl = P // 2, P // 2 // world
    rm = torch.stack([returns[:pairs].view(world, pl), returns[pairs:].view(world, pl)], 1).reshape(-1)
    out = []
    for r in range(world):
        part, ranks = be.zeros(n), be.zeros(P, dtype=torch.int32)
        k = (offs if key is None else key)[r * pl:(r + 1) * pl]
        so = order if world == 1 else torch.argsort(k, stable=True).to(torch.int32)
        be.rank_grad(rm if world > 1 else returns, None, 1.0, 0.0, P, table, offs[r * pl:(r + 1) * pl].contiguous(),
                     so.contiguous(), r * pl, pl, n, part, ranks, None, world=world)
        out += [ranks, part]
    return tuple(out)


def _returns(be, P, seed):
    ret = torch.randn(P, generator=torch.Generator().manual_seed(seed)).to(be.device)
    assert ret.unique().numel() == P
    return ret


@pytest.mark.parametrize("form", ["table", "table16"])
@pytest.mark.parametrize("fn,world", [("adam", 1), ("raw", 1), ("raw", 4)])
@pytest.mark.parametrize("n,P", [(4610, 4096), (1001760, 64)])
def test_rank_grad_relocated(be, big, n, P, fn, world, form):
    pairs = P // 2
    offs, order = offsets_of(be, n, pairs)
    ret = _returns(be, P, n + P)
    theta, m = randn(be, n, seed=22, scale=0.1), randn(be, n, seed=23, scale=0.01)
    v = randn(be, n, seed=24, scale=1e-3).abs()
    small, s16, _, soffs = relocate(big, offs, n)
    runs = {"big": (big.t16 if form == "table16" else big.t, offs),
            "small": (s16 if form == "table16" else small, soffs)}
    out = {name: _rank_grad(be, fn, ret, t, o, order, n, theta, m, v, world, key=offs)
           for name, (t, o) in runs.items()}
    assert len(out["big"]) == len(out["small"])
    for a, b in zip(out["big"], out["small"]):
        same_bits(a, b)


_WANT = {}


def _grad64(be, big, n, P, ret, offs):
    """float64 sum_j (c_j - c_{j+pairs}) * T[off_j : off_j + n] over the rows the offsets name (on the device,
    in chunks), and the ranks (stable argsort of the returns)."""
    key = (n, P)
    if key not in _WANT:
        pairs = P // 2
        ranks = torch.empty(P, dtype=torch.int64, device=be.device)
        ranks[torch.argsort(ret, stable=True)] = torch.arange(P, device=be.device)
        c = (ranks.double() / (P - 1) - 0.5).float()
        w = (c[:pairs] - c[pairs:]).double()
        acc = torch.zeros(n, dtype=torch.float64, device=be.device)
        idx = torch.arange(n, device=be.device)
        step = max(1, (1 << 24) // n)
        for j0 in range(0, pairs, step):
            acc += w[j0:j0 + step] @ big.t[offs[j0:j0 + step, None] + idx[None, :]].double()
        _WANT[key] = (ranks, acc)
    return _WANT[key]


@pytest.mark.parametrize("form", ["table", "table16"])
@pytest.mark.parametrize("fn", ["adam", "raw"])
@pytest.mark.parametrize("n", GRAD_N)
def test_rank_grad_vs_float64(be, big, n, fn, form):
    P = 4096
    offs, order = offsets_of(be, n, P // 2)
    ret = _returns(be, P, 99)
    theta, m = randn(be, n, seed=25, scale=0.1), randn(be, n, seed=26, scale=0.01)
    v = randn(be, n, seed=27, scale=1e-3).abs()
    t = big.t16 if form == "table16" else big.t
    out = _rank_grad(be, fn, ret, t, offs, order, n, theta, m, v)
    ranks_want, acc = _grad64(be, big, n, P, ret, offs)
    assert torch.equal(out[0].long(), ranks_want)
    if fn == "raw":
        got, want = out[1], acc
    else:
        got, want = out[1], acc / P
    err = float((got.double() - want).abs().max() / want.abs().max())
    print(f"n={n} {fn} {form}: gradient vs float64 {err:.2e}")
    assert err < 1e-5
    if fn == "adam":
        th, mm, vv = orc.adam_step(theta.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy(),
                                   orc.negate_clamp(out[1].cpu().numpy()), 1)
        assert rel_err(out[2].cpu().numpy(), th) < 1e-6
        assert rel_err(out[3].cpu().numpy(), mm) < 1e-6 and rel_err(out[4].cpu().numpy(), vv) < 1e-6


# ------------------------------------------------------------------ offsets at large table lengths
LENGTHS = [TABLE_LEN, 1 << 32, (1 << 33) + 96, _capi.ESTK_MAX_TABLE_LEN - 32, _capi.ESTK_MAX_TABLE_LEN]


@pytest.mark.parametrize("table_len", LENGTHS)
@pytest.mark.parametrize("pairs", [1000, 4096, 6000])
@pytest.mark.parametrize("n", [4610, 1001760])
def test_make_offsets_at_large_table_lengths(be, table_len, pairs, n):
    """No table is read: estk_make_offsets' offsets and order at table lengths up to ESTK_MAX_TABLE_LEN, bit-exact
    against the oracle's hash and the stable argsort, on the one-CTA sort (<= 4096 pairs) and the grid-wide sort."""
    seed, gen, begin = 0xDEADBEEF12345, 3, 256
    offs, order = be.alloc(pairs, dtype=torch.int64), be.alloc(pairs, dtype=torch.int32)
    be.make_offsets(seed, None, gen, begin, pairs, table_len, n, offs, order)
    want = orc.noise_offsets(seed, gen, begin, pairs, table_len, n)
    got = offs.cpu().numpy()
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(order.cpu().numpy(), np.argsort(want, kind="stable"))
    assert got.max() + ceil32(n) <= table_len and got.max() >= table_len // 2


def test_make_offsets_refuses_a_table_beyond_the_limit(be):
    offs = be.alloc(4, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="longer than"):
        be.make_offsets(1, None, 0, 0, 4, _capi.ESTK_MAX_TABLE_LEN + 32, 4610, offs)


# ------------------------------------------------------------------ the cross-GPU reduction
def test_rank_grad_xr_relocated_on_two_gpus(tmp_path):
    """estk_rank_grad_xr_adam on two GPUs, each with its own 2^31 + 2^22 entry table: the big table at the big
    offsets and the relocated small table give the same theta / m / v / gradient bits on both ranks."""
    if torch.cuda.device_count() < 2:
        pytest.skip("estk_rank_grad_xr_adam needs 2 GPUs; this host has fewer")
    for d in range(2):
        free, _ = torch.cuda.mem_get_info(d)
        if free < NEED_BYTES:
            pytest.skip(f"needs {NEED_BYTES / GIB:.1f} GiB free on GPU {d}; {free / GIB:.1f} GiB free")
    import socket
    import subprocess
    import sys
    import textwrap
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "xr_large_table.py"
    script.write_text(textwrap.dedent(f"""
        import os, sys
        sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
        import torch, torch.distributed as dist
        import test_large_table_gpu as T
        from estorch_b200.backend import CudaBackend, adam_desc, new_state
        rank, W = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
        dist.init_process_group("gloo")
        be = CudaBackend(torch.device("cuda", rank))
        big = T.Big(be)
        n, P = 4610, 4096
        pairs = P // 2
        pl = pairs // W
        offs, order = T.offsets_of(be, n, pairs)
        ret = T._returns(be, P, 5)
        rm = torch.stack([ret[:pairs].view(W, pl), ret[pairs:].view(W, pl)], 1).reshape(-1).contiguous()
        theta = T.randn(be, n, seed=28, scale=0.1)
        mine = be.peer_alloc(be.xr_workspace_bytes(n))
        handles = [None] * W
        dist.all_gather_object(handles, mine[1])
        ptrs = [mine[0] if r == rank else be.peer_open(handles[r]) for r in range(W)]
        small, s16, _, soffs = T.relocate(big, offs, n)
        out = {{}}
        for name, t16, o in (("big", big.t16, offs), ("small", s16, soffs)):
            lo = o[rank * pl:(rank + 1) * pl].contiguous()
            so = torch.argsort(offs[rank * pl:(rank + 1) * pl], stable=True).to(torch.int32)   # the same order
            th, m, v, g = theta.clone(), be.zeros(n), be.zeros(n), be.zeros(n)
            dist.barrier()
            be.rank_grad_xr_adam(rm, None, 1.0, 0.0, P, W, rank, t16, lo, so, rank * pl, pl, ptrs, th, m, v,
                                 new_state(be.device), adam_desc(lr=0.01), None, None, g)
            torch.cuda.synchronize()
            out[name] = (th, m, v, g)
        for a, b in zip(out["big"], out["small"]):
            T.same_bits(a, b)
        dist.barrier()
        be.peer_close_all()
        dist.barrier()
        be.peer_free_all()
        print("xr relocated ok")
        dist.destroy_process_group()
    """))
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    assert r.stdout.count("xr relocated ok") == 2
