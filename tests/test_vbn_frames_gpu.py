"""The conv + VirtualBatchNorm kernels on Atari-like frames (tests/_vbn_frames.py: raw 0..255 pixels, constant
backgrounds, near-zero and zero variances, a reference frame that is an outlier) against a float64 forward of the
same members.

The tensor-core ("f16") evaluate's returns are checked on every frame kind both at 0..255 and divided by 255.

Bar: max-norm relative error (per member) below max(1e-5, k e_ref), e_ref the reference fp32 forward's own error on
the same quantity and inputs (the policy in torch float32 on the CPU).  The VBN scales a = gamma / sqrt(var + 1e-5)
are compared element by element.  Where a pixel never changes over the reference batch, a is ~300 and a fp32 conv
output's rounding is already ~1e-3 of a normalised value, so no fp32 implementation meets a flat 1e-5 there; e_ref
says how far the reference's own fp32 arithmetic gets.  k = 4 for the returns of a population-mode ES generation.
For the statistics, outputs and returns of single members k depends on R (K_MEMBER), about twice the worst the
kernels measured on an H100: up to 8 e_ref at R <= 8, up to 69 e_ref at R = 128 (a2 on outlier frames, from the
layer-2 statistics; layer 1 stays within ~2 e_ref).  The one-pass variance the fp32 kernels used before is off by
a relative 1 to 80 in a at R >= 8 (tests/test_vbn_frames_cpu.py), beyond 1e4 e_ref."""
import numpy as np
import pytest
import torch

import _vbn_frames as vf
from oracle import es_oracle as orc
from _pop_conv_oracle import STATS_FLOATS, AtariPolicy, PixelWalker

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA GPU", allow_module_level=True)

import estorch_b200 as E  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402

f32, f64 = np.float32, np.float64
PAIRS, SIGMA = 2, 0.02
K_MEMBER = {2: 16, 3: 16, 8: 16, 128: 100}


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _bar(e_ref, k=4):
    return max(1e-5, k * e_ref)


def _eval_return(y, t):
    """The fp32 evaluate's return from one member's outputs y [B, A], B <= 32: thread k accumulates
    fmaf(d, d, .) over elements k, k + 256, ...; warp_sum_f's xor butterfly; the 8 warps in order."""
    d = (y - t).astype(f32).reshape(-1)
    v = np.zeros(256, dtype=f32)
    for k0 in range(0, d.size, 256):
        e = d[k0:k0 + 256]
        v[:e.size] = orc.fma32(e, e, v[:e.size])
    v = v.reshape(8, 32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[:, lanes ^ o]).astype(f32)
    s = f32(0)
    for w in range(8):
        s = f32(s + v[w, 0])
    return -(s / (f32(y.shape[0]) * f32(y.shape[1])))


def _cases():
    out = []
    for ki, kind in enumerate(vf.KINDS):
        for ri, R in enumerate((2, 3, 8, 128)):
            out.append((kind, R, (1, 3, 32)[(ki + ri) % 3], (4, 18)[(ki + ri // 2) % 2],
                        ("init", "trained")[(ki + ri) % 2]))
    return out


def _d(be, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(be.device)


def _oracle(rows, A, xref, obs, tgt):
    """Float64 and reference-fp32 outputs, statistics and returns of every member row."""
    want_out, want_st, ref_out, ref_st = [], [], [], []
    for row in rows:
        f = vf.Forward64(row, A, xref)
        want_out.append(f(obs))
        want_st.append(f.folded())
        o32, s32 = vf.reference32(row, A, xref, obs)
        ref_out.append(o32)
        ref_st.append(s32)
    want_ret = np.array([-np.mean((o - tgt) ** 2) for o in want_out])
    ref_ret = np.array([-np.mean((o - tgt) ** 2) for o in ref_out])
    return want_out, want_st, want_ret, ref_out, ref_st, ref_ret


@pytest.mark.parametrize("kind,R,B,A,theta", _cases(), ids=lambda v: str(v))
def test_vbn_kernels_against_float64(be, kind, R, B, A, theta):
    seed = 1000 * R + 10 * B + A
    row = vf.policy_row(A, theta, seed)
    n = row.size
    rng = np.random.RandomState(seed)
    table = orc.round_f16(rng.standard_normal((n + 31) // 32 * 32 + 4096).astype(f32))
    offs = orc.noise_offsets(seed, 0, 0, PAIRS, table.size, n)
    xref, obs = vf.frames(kind, R, B, seed=seed)
    tgt = rng.standard_normal((B, A)).astype(f32)
    rows = np.concatenate([orc.sample_population(row, table, offs, SIGMA)[0], row[None]])   # + members, -, centre
    M = rows.shape[0]

    want_out, want_st, want_ret, ref_out, ref_st, ref_ret = _oracle(rows, A, xref, obs, tgt)

    # ---- the kernels: stats + act (population and centre), fp32 and f16 evaluate, each twice
    th, tb, of, xr, ob, tg = (_d(be, a) for a in (row, table, offs, xref, obs, tgt))
    tb16 = tb.to(torch.float16)

    def act():
        st, out = be.alloc(2 * PAIRS, STATS_FLOATS), be.alloc(2 * PAIRS, B, A)
        be.act_conv_vbn(A, th, tb, of, None, PAIRS, SIGMA, xr, ob[None].expand(2 * PAIRS, B, 4, 84, 84).contiguous(),
                        out, st)
        stc, outc = be.alloc(1, STATS_FLOATS), be.alloc(1, B, A)
        be.act_conv_vbn(A, th, None, None, None, 1, 0.0, xr, ob[None], outc, stc)
        return torch.cat([st, stc]).cpu().numpy(), torch.cat([out, outc]).cpu().numpy()

    def evaluate(precision, xr=xr, ob=ob):
        scratch = torch.empty(be.conv_scratch_bytes(R, B, precision), dtype=torch.uint8, device=be.device)
        r = be.zeros(2 * PAIRS + 1)
        kw = {"table16": tb16} if precision == "f16" else {}
        be.eval_conv_vbn(A, th, tb, of, None, PAIRS, SIGMA, xr, ob, tg, r[:PAIRS], r[PAIRS:2 * PAIRS], scratch,
                         precision=precision, **kw)
        be.eval_conv_vbn(A, th, None, None, None, 1, 0.0, xr, ob, tg, r[2 * PAIRS:], None, scratch,
                         precision=precision)
        return r.cpu().numpy()

    st, out = act()
    ret32 = evaluate("fp32")
    st2, out2 = act()
    assert np.array_equal(st.view(np.uint32), st2.view(np.uint32))           # the same bits run to run
    assert np.array_equal(out.view(np.uint32), out2.view(np.uint32))
    assert np.array_equal(evaluate("fp32").view(np.uint32), ret32.view(np.uint32))

    # ---- act mode's outputs are the bits of the fp32 evaluate's
    got = np.array([_eval_return(out[m], tgt) for m in range(M)], dtype=f32)
    assert np.array_equal(got.view(np.uint32), ret32.view(np.uint32)), (got, ret32)

    # ---- statistics, outputs and returns against float64
    report = []
    for m in range(M):
        for name, sl in vf.stats_slices():
            err = vf.scale_err if name[0] == "a" else vf.rel_err
            e, e_ref = err(st[m, sl], want_st[m][sl]), err(ref_st[m][sl], want_st[m][sl])
            report.append((f"member {m} {name}", e, e_ref))
        report.append((f"member {m} outputs", vf.rel_err(out[m], want_out[m]), vf.rel_err(ref_out[m], want_out[m])))
    e_ref = vf.rel_err(ref_ret, want_ret)
    report.append(("fp32 evaluate returns", vf.rel_err(ret32, want_ret), e_ref))
    ret16 = evaluate("f16")
    assert np.array_equal(evaluate("f16").view(np.uint32), ret16.view(np.uint32))
    report.append(("f16 evaluate returns", vf.rel_err(ret16, want_ret), e_ref))
    if kind != "unit":      # the same frames divided by 255
        xs, os_ = (xref / f32(255)).astype(f32), (obs / f32(255)).astype(f32)
        want_s, ref_s = _oracle(rows, A, xs, os_, tgt)[2::3]
        ret16 = evaluate("f16", _d(be, xs), _d(be, os_))
        report.append(("f16 evaluate returns, frames / 255", vf.rel_err(ret16, want_s), vf.rel_err(ref_s, want_s)))
    k = K_MEMBER[R]
    bad = [(what, f"{e:.2e}", f"bar {_bar(r, k):.2e}") for what, e, r in report if not e < _bar(r, k)]
    worst = max(report, key=lambda t: t[1] / max(2.5e-6, t[2]))
    print(f"{kind} R={R} B={B} A={A} {theta}: worst {worst[0]} {worst[1]:.2e}, "
          f"{worst[1] / max(2.5e-6, worst[2]):.1f} x max(2.5e-6, e_ref); {len(bad)} over the bar of {k} e_ref")
    assert not bad, bad


# ------------------------------------------------------------------ the engine: population-mode ES on raw frames
class RawWalker(PixelWalker):
    """PixelWalker rendered like an Atari screen: a bright blob (up to 255) on a constant grey background (142)."""
    GAIN = 2e-5             # logits of raw-scale frames reach ~1e4

    def frames(self, s):
        g = (torch.arange(84, device=s.device, dtype=torch.float32) + 0.5) / 42.0 - 1.0
        d2 = (g[None, :, None] - s[:, 0, None, None]) ** 2 + (g[None, None, :] - s[:, 1, None, None]) ** 2
        w = torch.tensor(self.WIDTHS, device=s.device, dtype=torch.float32)
        blob = torch.exp(-d2[:, None] / (2 * w * w)[None, :, None, None])
        return (vf.BG + (vf.BRIGHT - vf.BG) * blob).float().contiguous()


def _raw_xref(R=8, seed=3):
    g = torch.Generator().manual_seed(seed)
    pts = (0.3 * torch.randn(R, 2, generator=g)).clamp(-0.9, 0.9)
    return RawWalker().frames(pts)


def test_population_es_on_raw_frames_against_float64():
    A, P, horizon = 4, 16, 4
    xref = _raw_xref()
    rec = {}

    class Q(E.ES):
        def log(self):
            rec["returns"] = self.population_returns[:, 0].copy()
            rec["theta"] = self._slots[0].theta_prev.cpu().numpy().copy()
            rec["offsets"] = self._offsets.cpu().numpy().copy()
    torch.manual_seed(0)
    es = Q(AtariPolicy, RawWalker, torch.optim.Adam, population_size=P, sigma=0.02,
           policy_kwargs={"n_actions": A, "xref": xref}, agent_kwargs={"horizon": horizon},
           optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 21, noise_seed=5)
    assert es._population and es._is_conv and es._precision == "fp32"
    es.train(n_steps=1)
    rows, _ = orc.sample_population(rec["theta"], es._table.cpu().numpy(), rec["offsets"], 0.02)
    xr = xref.numpy()

    def rollout(forward):
        """Every member's return with forward(m, frames [1, 4, 84, 84] fp32) -> outputs [1, A] in float64."""
        def act(frames):
            x = frames.float().numpy()
            return torch.from_numpy(np.concatenate([forward(m, x[m:m + 1]) for m in range(P)]))
        return RawWalker(horizon=horizon).rollout_population(act, P).numpy()

    fwd64 = [vf.Forward64(r, A, xr) for r in rows]
    want = rollout(lambda m, x: fwd64[m](x))
    ref = rollout(lambda m, x: vf.reference32(rows[m], A, xr, x)[0])
    e, e_ref = vf.rel_err(rec["returns"], want), vf.rel_err(ref, want)
    print(f"population ES on raw frames: returns {e:.2e} from float64, reference fp32 {e_ref:.2e}")
    assert e < _bar(e_ref)
