"""The Atari-like VirtualBatchNorm frames and the float64 forward of tests/_vbn_frames.py, without a GPU: the
float64 forward is the policy's own arithmetic (a torch float64 run agrees to ~1e-12), and the frames tell an
accurate variance from the one-pass sum-of-squares formula the fp32 kernels used to compute, while uniform random
frames, what every other conv test feeds, do not."""
import numpy as np
import pytest
import torch

import _vbn_frames as vf
from _pop_conv_oracle import AtariPolicy

R = 8
_row = vf.policy_row


def test_frames_are_deterministic_and_atari_like():
    for kind in vf.KINDS:
        xref, obs = vf.frames(kind, 5, 3, seed=4)
        xref2, obs2 = vf.frames(kind, 5, 3, seed=4)
        assert xref.dtype == obs.dtype == np.float32 and xref.shape == (5, 4, 84, 84) and obs.shape == (3, 4, 84, 84)
        assert np.array_equal(xref, xref2) and np.array_equal(obs, obs2)
        top = 1.0 if kind == "unit" else 255.0
        assert xref.min() >= 0 and xref.max() <= top and xref.max() > 0.5 * top
        const = (xref == xref[:1]).all(0)
        assert const.mean() > 0.5, kind                        # most pixels never change over the batch
        assert (obs != xref[:1])[:, const].any(), kind          # observations differ where the batch is constant
    xref, _ = vf.frames("same", 4, 1)
    assert (xref == xref[:1]).all()
    xref, _ = vf.frames("outlier", 4, 1)
    assert (xref[1:] == xref[1:2]).all() and (xref[0] != xref[1]).any()


@pytest.mark.parametrize("kind", ["raw", "near", "outlier"])
def test_float64_forward_is_the_policy_in_float64(kind):
    A = 4
    row = _row(A, "trained", 3)
    xref, obs = vf.frames(kind, R, 3, seed=1)
    f = vf.Forward64(row, A, xref)
    pol = AtariPolicy(A, torch.from_numpy(xref).double()).double()
    torch.nn.utils.vector_to_parameters(torch.from_numpy(row).double(), pol.parameters())
    with torch.no_grad():
        want = pol(torch.from_numpy(obs).double()).numpy()
        F = torch.nn.functional
        F.relu(pol.bn2(pol.conv2(F.relu(pol.bn1(pol.conv1(pol.xref))))))
        stats = [(bn.mean.numpy(), bn.var.numpy()) for bn in (pol.bn1, pol.bn2)]
    assert vf.rel_err(f(obs), want) < 1e-12
    for (m, v), (tm, tv) in zip(f.stats, stats):
        assert vf.rel_err(m, tm) < 1e-12 and vf.rel_err(v, tv) < 1e-12


@pytest.mark.parametrize("kind", list(vf.KINDS) + ["rand"])
def test_one_pass_variance_misses_the_bar_where_welford_meets_it(kind):
    """Layer 1's scale a = gamma / sqrt(var + 1e-5) from the fp32 kernels' conv1 (one fmaf chain per output),
    against float64.  The bar is the one the GPU tests use: max(1e-5, 4 e_ref), e_ref the reference fp32
    forward's error on the same statistic.  Welford's update meets it on every frame kind; the one-pass
    (ssq - sum * mean) / (R - 1) meets it only on uniform random frames."""
    A = 4
    row = _row(A, "init", 7)
    if kind == "rand":
        g = torch.Generator().manual_seed(2)
        xref, obs = torch.rand(R, 4, 84, 84, generator=g).numpy(), torch.rand(2, 4, 84, 84, generator=g).numpy()
    else:
        xref, obs = vf.frames(kind, R, 2, seed=2)
    want = vf.Forward64(row, A, xref).folded()[:vf.P1]
    _, ref32 = vf.reference32(row, A, xref, obs)
    bar = max(1e-5, 4 * vf.scale_err(ref32[:vf.P1], want))
    y = vf.conv1_fp32_chain(xref, row[:4096].reshape(16, 4, 8, 8), row[4096:4112])
    gamma = row[4112:4128]
    e_one = vf.scale_err(vf.vbn1_scale_one_pass(y, gamma).reshape(-1), want)
    e_welford = vf.scale_err(vf.vbn1_scale_welford(y, gamma).reshape(-1), want)
    print(f"{kind}: one-pass {e_one:.2e}, Welford {e_welford:.2e}, bar {bar:.2e}")
    assert e_welford < bar
    if kind == "rand":
        assert e_one < bar
    else:
        assert e_one > 10 * bar
