"""The float64 restatement of the 16-bit tensor-core MLP evaluate (tests/_tc_mlp_model.py) on the CPU: it agrees with
the oracle's emulations, its bound holds for a restatement that accumulates in fp32 blocks of 16 with truncation,
and the bound is tight enough that each of the faults a warp-specialised kernel can make in one tile, one stage or
one sign breaks it for some output."""
import numpy as np
import pytest
import torch

import _mlp_oracle as mlp
import _tc_mlp_model as tcm
from oracle import es_oracle as orc

# shapes of tests/test_eval_mlp_tc_bounds_gpu.py, at a CPU-sized batch
SHAPES = {"one_layer": [64, 32], "widest_f16": [256, 512, 512, 512], "bf16_wide_in": [512, 512, 32],
          "eight_narrow": [64] * 8 + [32], "odd_tiles": [128, 384, 160]}
B = 64


def problem(dims, pairs=2, seed=3, w_scale=1.0, obs_scale=1.0):
    rng = np.random.RandomState(seed)
    n = orc.mlp_param_count(dims)
    table_len = (n + 31) // 32 * 32 + (1 << 12)
    table = orc.round_f16(rng.standard_normal(table_len).astype(np.float32))
    theta = np.concatenate([np.concatenate([rng.uniform(-1, 1, k * m), rng.uniform(-1, 1, m)]) * w_scale / np.sqrt(k)
                            for k, m in zip(dims[:-1], dims[1:])]).astype(np.float32)
    obs = (rng.standard_normal((B, dims[0])) * obs_scale).astype(np.float32)
    offs = orc.noise_offsets(11, 0, 0, pairs, table_len, n)
    return theta, table, obs, offs


def trunc32(x):
    """float64 -> fp32 rounded toward zero, as float64."""
    r = tcm.fl32(x)
    over = r.abs() > x.abs()
    return torch.where(over, torch.nextafter(r.to(torch.float32), torch.zeros_like(r, dtype=torch.float32))
                       .to(torch.float64), r)


def restate(mode, rows, dims, ops, code, drop_kblock=None):
    """The kernel's order of operations: per N tile, k-blocks of 64 in ascending order (layer 0 in fp16: the x_hi then
    the x_lo k-block on the same weights), each as four k16 MMAs whose exact sums enter the fp32 accumulator rounded
    toward zero; + bias in fp32; the fp32 activation (``orc.HIDDEN``); rounded once to 16 bits.  ``drop_kblock`` =
    (layer, tile, kb) skips that stage."""
    hidden, output, _ = mlp.decode(code)
    M = rows.shape[0]
    for li, (K, N, ws, bs) in enumerate(tcm.layout(dims)):
        W = rows[:, ws].reshape(M, N, K).transpose(1, 2)
        acc = torch.zeros(M, ops[0].shape[-2], N, dtype=torch.float64)
        for kb in range(0, K, 64):
            for o in ops:
                for k16 in range(kb, min(kb + 64, K), 16):
                    part = o[..., k16:k16 + 16] @ W[:, k16:k16 + 16]
                    if drop_kblock is not None and drop_kblock[:2] == (li, 0) and drop_kblock[2] == kb // 64:
                        part[..., :128] = 0
                    acc = trunc32(acc + part)
        y = tcm.fl32(acc + rows[:, bs][:, None, :])
        if li == len(dims) - 2:
            return tcm.t64(np.tanh(y.numpy().astype(np.float32))) if output == "tanh" else y
        a = torch.from_numpy(orc.HIDDEN[hidden](y.numpy().astype(np.float32)).astype(np.float64))
        ops = [tcm.rn16(a, tcm.kind(mode))]


def ratio(got, y, bound):
    return float(((got - y).abs() / bound.clamp(min=1e-300)).max())


# ------------------------------------------------------------------ agreement with the oracle's emulations
@pytest.mark.parametrize("mode", ["f16", "bf16", "bf16s"])
def test_model_matches_oracle_emulation_except_counted_formation_flips(mode):
    dims, sigma = [128, 256, 64], 0.02
    theta, table, obs, offs = problem(dims, pairs=4)
    rows = tcm.form(mode, dims, theta, table, offs, sigma)
    if mode == "bf16s":
        ref = tcm.t64(orc.sample_population_bf16s(theta, table, offs, sigma))
    else:
        pop, _ = orc.sample_population(theta, table, offs, sigma)
        ref = tcm.rn16(tcm.t64(pop), tcm.kind(mode))
    w = tcm.is_weight(dims)
    flips = (rows != ref) & w[None]
    # a flip is one 16-bit spacing, or the oracle's rounding of sigma * eps where theta and it nearly cancel
    room = torch.maximum(tcm.spacing(rows, tcm.kind(mode)), tcm.spacing(ref, tcm.kind(mode))) + \
        2 * tcm.U32 * (rows - tcm.t64(theta)[None]).abs()
    n_flip = int(flips.sum())
    print(f"{mode}: {n_flip} of {int(w.sum()) * rows.shape[0]} weights differ from the oracle's two roundings")
    assert n_flip < 1e-3 * int(w.sum()) * rows.shape[0]
    assert bool(((rows - ref).abs()[flips] <= room[flips]).all())
    # biases: the oracle rounds sigma * eps, then the sum; the kernel one fma -- both within an ulp
    assert float(((rows - tcm.t64(orc.sample_population(theta, table, offs, sigma)[0]))[:, ~w]).abs().max()) < 1e-6
    # the oracle's forward on its own weights lies within the model's bound of the model on those weights
    ops = tcm.layer0(mode, obs)
    ref_rows = torch.where(w[None], ref, rows)
    y, bound, _ = tcm.forward(mode, ref_rows, dims, ops, 0)
    fwd = orc.mlp_forward_f16 if tcm.kind(mode) == "f16" else orc.mlp_forward_bf16
    emu = torch.stack([tcm.t64(fwd(ref_rows[i].numpy().astype(np.float32), dims, obs)) for i in range(len(rows))])
    assert ratio(emu, y, bound) <= 1.0


def test_rn16_matches_numpy_and_satfinite():
    x = np.concatenate([np.random.RandomState(0).standard_normal(4096) * 10.0 ** np.arange(-8, 8).repeat(256),
                        [0.0, 65504.0, 65519.0, 65520.0, 1e6, np.inf, -np.inf, 2.0 ** -25, 3 * 2.0 ** -26]])
    x32 = x.astype(np.float32)
    got = tcm.rn16(tcm.t64(x32), "f16").numpy()
    np.testing.assert_array_equal(got, orc.round_f16(x32).astype(np.float64))
    np.testing.assert_array_equal(tcm.rn16(tcm.t64(x32), "bf16").numpy(), orc.round_bf16(x32).astype(np.float64))
    a, b, c = (np.random.RandomState(i).standard_normal(1 << 14).astype(np.float32) for i in range(3))
    np.testing.assert_array_equal(tcm.fma32(tcm.t64(a), tcm.t64(b), tcm.t64(c)).numpy(),
                                  orc.fma32(a, b, c).astype(np.float64))


def test_layer0_split_passes_infinities():
    """x_hi saturates and x_lo does not: a finite |x| keeps ~22 bits up to 131008, and +-inf or |x| >= 131024 enters
    with x_lo = +-inf, so its outputs are not finite."""
    x = np.array([[1.0, np.inf, -np.inf, np.nan, 1e6, 70000.0, 1 + 2.0 ** -20, 2.0 ** -30, 131023.0, -131024.0]],
                 np.float32)
    hi, lo = (o.numpy()[0] for o in tcm.layer0("f16", x))
    assert hi[1] == 65504 and lo[1] == np.inf and hi[2] == -65504 and lo[2] == -np.inf
    assert np.isnan(hi[3]) and np.isnan(lo[3])
    assert lo[4] == np.inf and hi[8] + lo[8] == 131008.0 and lo[9] == -np.inf
    assert hi[5] + lo[5] == 70000.0
    assert hi[6] == 1.0 and lo[6] == 2.0 ** -20
    assert hi[7] == 0.0 and lo[7] == 0.0


# ------------------------------------------------------------------ the bound holds for a truncating fp32 kernel
CASES = [(s, mode, code, dom) for s in SHAPES for mode in ("f16", "bf16", "bf16s")
         for code, dom in ((0, "1x"), (mlp.code("silu", "tanh"), "8x"), (mlp.code("tanh", loss="xent"), "x255"))
         if not (mode == "f16" and s == "bf16_wide_in")]
CASES += [("odd_tiles", "f16", c, "1x") for c in mlp.CODES]
DOMAINS = {"1x": (1.0, 1.0), "8x": (8.0, 1.0), "x255": (1.0, 255.0)}


@pytest.mark.parametrize("shape,mode,code,dom", CASES)
def test_bound_holds_for_truncating_fp32_restatement(shape, mode, code, dom):
    dims = SHAPES[shape]
    w_scale, obs_scale = DOMAINS[dom]
    theta, table, obs, offs = problem(dims, pairs=1, w_scale=w_scale, obs_scale=obs_scale)
    rows = tcm.form(mode, dims, theta, table, offs, 0.05, centre=True)
    ops = tcm.layer0(mode, obs)
    y, bound, exposed = tcm.forward(mode, rows, dims, ops, code)
    got = restate(mode, rows, dims, ops, code)
    r = ratio(got, y, bound)
    print(f"{shape} {mode} {code:#x} {dom}: worst error / bound {r:.3f}, exposed {int(exposed.sum())}")
    assert torch.isfinite(y).all() and r <= 1.0


# ------------------------------------------------------------------ detection power
# Tile-local faults go into the last layer, where nothing rounds them away.  A worst-case bound loosens with every
# 16-bit hidden layer in front of an output: each layer may flip the roundings of the inputs whose error interval
# reaches a boundary, and the flips' intervals grow from layer to layer.  Behind eight hidden layers, or three of 512
# inputs for a fault as small as one missing bias tile, it no longer separates faults of an output's own size; the
# operand faults (x_lo dropped, bf16 rounding in fp16 mode: 2^-12 .. 2^-9 of each term, random signs) already hide
# behind one wide hidden layer.  Each fault is checked on the shapes where the bound sees it; the operand faults are
# also pinned bit for bit by the one-hot and identity-weight tests of tests/test_eval_mlp_tc_bounds_gpu.py.
MUTATIONS = {"drop_kblock": ["one_layer", "widest_f16", "bf16_wide_in", "odd_tiles"],
             "bias_tile": ["one_layer", "bf16_wide_in", "odd_tiles"],
             "wrong_sign": ["one_layer", "widest_f16", "bf16_wide_in", "odd_tiles"],
             "stale_stage": ["widest_f16", "bf16_wide_in", "odd_tiles"],
             "drop_xlo": ["one_layer"], "bf16_in_f16": ["one_layer", "odd_tiles"]}


def mutated(mutation, mode, dims, theta, table, offs, obs, sigma):
    """The restatement with one fault, on member 0 (sign +) or, for the operand faults, on every member."""
    rows = tcm.form(mode, dims, theta, table, offs, sigma)
    ops = tcm.layer0(mode, obs)
    P = len(offs)
    lay = tcm.layout(dims)
    last = len(lay) - 1
    if mutation == "drop_kblock":                  # the last layer's k-block 0 of N tile 0
        return restate(mode, rows, dims, ops, 0, drop_kblock=(last, 0, 0))
    if mutation == "drop_xlo":
        return restate(mode, rows, dims, ops[:1], 0)
    rows = rows.clone()
    K, N, ws, bs = lay[last]
    if mutation == "bias_tile":                    # the last layer's last N tile without its bias
        rows[0, bs.start + (N - 1) // 128 * 128: bs.stop] = 0
    elif mutation == "stale_stage":                # tile 1's k-block 0 formed as tile 0's (a layer with two tiles)
        K, N, ws, _ = next(x for x in reversed(lay) if x[1] > 128)
        W = rows[0, ws].view(N, K)
        W[128:256, :64] = W[0:128, :64][: min(N, 256) - 128]
    elif mutation == "wrong_sign":                 # the last layer's tile 0 formed with the other sign
        rows[0, ws].view(N, K)[:128] = rows[P, ws].view(N, K)[:128]
    elif mutation == "bf16_in_f16":
        rows = tcm.form("bf16", dims, theta, table, offs, sigma)
    return restate(mode, rows, dims, ops, 0)


@pytest.mark.parametrize("mutation,shape", [(m, s) for m, shapes in MUTATIONS.items() for s in shapes])
def test_every_fault_breaks_the_bound(mutation, shape):
    dims = SHAPES[shape]
    mode = "bf16" if shape == "bf16_wide_in" else "f16"
    sigma = 0.05
    theta, table, obs, offs = problem(dims, pairs=1)
    rows = tcm.form(mode, dims, theta, table, offs, sigma)
    y, bound, _ = tcm.forward(mode, rows, dims, tcm.layer0(mode, obs), 0)
    clean = restate(mode, rows, dims, tcm.layer0(mode, obs), 0)
    assert ratio(clean, y, bound) <= 1.0
    bad = mutated(mutation, mode, dims, theta, table, offs, obs, sigma)
    r = ratio(bad, y, bound)
    print(f"{shape} {mutation}: worst error / bound {r:.1f}")
    assert r > 1.0, f"{mutation} stays within the bound on {dims}"
