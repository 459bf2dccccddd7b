"""Tensor-core evaluate: tile ownership between the two consumer warpgroups.

The N tiles of every CTA's (task, layer, N tile) sequence alternate between two consumer
warpgroups, so results depend on the tile-order handoff, the per-layer barriers and the loss
chain handed from one warpgroup to the other in the last layer.  These shapes put 1..4 N tiles
(and a narrow last tile) in the last layer, a single tile in a hidden layer, odd and even tile
counts per task, two clusters per sign (B = 512), and enough pairs that every CTA runs several
tasks, so a warpgroup's first tile of a task is sometimes tile 0 and sometimes not.
"""
import numpy as np
import pytest
import torch

from oracle import es_oracle as orc
from conftest import rel_err

pytestmark = pytest.mark.gpu

# (dims, B, pairs, bc): tiles per task = sum over layers of ceil(N / 128)
SHAPES = [
    ([64, 128, 32], 256, 48, 0),          # 2 tiles per task, narrow single last tile
    ([64, 128, 160], 256, 48, 256),       # 3: last layer 128 + 32, with BC
    ([128, 256, 256], 256, 40, 0),        # 4: two tiles in each layer
    ([64, 128, 288], 512, 24, 0),         # 4, two clusters per sign
    ([128, 512, 128, 416], 256, 40, 64),  # 9: single-tile hidden layer, last 3 x 128 + 32
    ([64, 128, 512], 256, 48, 0),         # 5: last layer 4 full tiles
]
TOL = {"f16": 1e-5, "bf16": 5e-4, "bf16s": 5e-4}


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def dev(be, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(be.device)


def _problem(dims, B, pairs, seed=5):
    rng = np.random.RandomState(seed)
    n = orc.mlp_param_count(dims)
    table_len = (n + 31) // 32 * 32 + (1 << 14)
    table = orc.round_f16(rng.standard_normal(table_len).astype(np.float32))
    theta = np.concatenate([np.concatenate([(rng.uniform(-1, 1, dims[i] * dims[i + 1]) / np.sqrt(dims[i])),
                                            rng.uniform(-1, 1, dims[i + 1]) / np.sqrt(dims[i])])
                            for i in range(len(dims) - 1)]).astype(np.float32)
    obs = rng.standard_normal((B, dims[0])).astype(np.float32)
    tgt = rng.standard_normal((B, dims[-1])).astype(np.float32)
    offs = orc.noise_offsets(11, 0, 0, pairs, table_len, n)
    return n, table, theta, obs, tgt, offs


def _bf16s_rows(theta, table, offs, dims, sigma):
    """Rows as the bf16s mode forms them: weights from bf16 shadows, biases from fp32 sources."""
    exact, _ = orc.sample_population(theta, table, offs, sigma)
    rows = orc.sample_population_bf16s(theta, table, offs, sigma)
    centre = orc.round_bf16(theta).copy()
    idx = 0
    for i in range(len(dims) - 1):
        idx += dims[i] * dims[i + 1]
        rows[:, idx: idx + dims[i + 1]] = exact[:, idx: idx + dims[i + 1]]
        centre[idx: idx + dims[i + 1]] = theta[idx: idx + dims[i + 1]]
        idx += dims[i + 1]
    return rows, centre


@pytest.mark.parametrize("mode", ["f16", "bf16", "bf16s"])
@pytest.mark.parametrize("dims,B,pairs,bc", SHAPES)
def test_tile_ownership_returns_bc_and_folded_centre(be, mode, dims, B, pairs, bc):
    sigma = 0.02
    n, table, theta, obs, tgt, offs = _problem(dims, B, pairs)
    assert be.eval_supports_f16(dims, B) and be.eval_supports_bf16(dims, B)
    order = np.argsort(offs, kind="stable").astype(np.int32)
    th, tb = dev(be, theta), dev(be, table)
    kw, ckw = {}, {}
    if mode == "f16":
        tb16 = be.alloc(table.size, dtype=torch.float16)
        assert be.shadow_f16(tb, tb16) == 0
        kw = {"table16": tb16}
    elif mode == "bf16s":
        th16 = be.alloc(n, dtype=torch.bfloat16)
        tb16 = be.alloc(table.size, dtype=torch.bfloat16)
        be.shadow_bf16(th, th16)
        be.shadow_bf16(tb, tb16)
        kw = {"theta16": th16, "table16": tb16}
        ckw = {"theta16": th16}
    obs_d, tgt_d, offs_d, order_d = dev(be, obs), dev(be, tgt), dev(be, offs), dev(be, order)

    def launch():
        ret, centre = be.zeros(2 * pairs), be.zeros(1)
        bcp = be.zeros(pairs, bc) if bc else None
        bcm = be.zeros(pairs, bc) if bc else None
        be.eval_mlp(dims, th, tb, offs_d, order_d, pairs, sigma, obs_d, tgt_d, ret[:pairs], ret[pairs:],
                    bcp, bcm, 64 if bc else 0, bc, precision=mode, centre_out=centre, **kw)
        torch.cuda.synchronize()
        out = [ret.cpu().numpy(), centre.cpu().numpy()]
        if bc:
            out.append(np.concatenate([bcp.cpu().numpy(), bcm.cpu().numpy()]))
        return out

    first, second = launch(), launch()
    for a, b in zip(first, second):                     # no atomics in the sums: same bits every launch
        np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))
    got, got_centre = first[0], first[1]

    # returns against the oracle's emulation of the mode's roundings
    if mode == "bf16s":
        rows, centre_row = _bf16s_rows(theta, table, offs, dims, sigma)
    else:
        rows, _ = orc.sample_population(theta, table, offs, sigma)
        centre_row = theta
    fwd = orc.mlp_forward_f16 if mode == "f16" else orc.mlp_forward_bf16
    outs = [fwd(rows[i], dims, obs) for i in range(2 * pairs)]
    emu = np.array([orc.synthetic_return(o, tgt) for o in outs], dtype=np.float32)
    assert rel_err(got, emu) < TOL[mode]
    want_centre = float(orc.synthetic_return(fwd(centre_row, dims, obs), tgt))
    assert abs(float(got_centre[0]) - want_centre) < TOL[mode] * abs(want_centre)

    # the folded centre task is the centre evaluation, bit for bit
    one = be.zeros(1)
    be.eval_mlp_center(dims, th, obs_d, tgt_d, one, precision=mode, **ckw)
    torch.cuda.synchronize()
    assert float(one) == float(got_centre[0])

    if bc:
        ref = orc.mlp_forward if mode == "f16" else fwd
        want_bc = np.stack([orc.synthetic_bc(ref(rows[i], dims, obs), 64, bc) for i in range(2 * pairs)])
        tol = 2e-3 if mode == "f16" else 5e-3
        assert np.max(np.abs(first[2] - want_bc)) < tol * np.max(np.abs(want_bc))
