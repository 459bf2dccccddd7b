"""The fused Adam step on the device, bit for bit against the oracle's restatement of torch.optim.Adam
(oracle/es_oracle.py ``adam_step``, itself held to torch in tests/test_adam_parity_cpu.py).

``adam_elem`` is the one function behind ``estk_clamp_adam``, ``estk_rank_grad_adam`` and
``estk_rank_grad_xr_adam``.  Given the kernel's own gradient bits (``grad_out``), theta / m / v after the
step must be the oracle's Adam of those bits exactly -- over the hyperparameter grid, every rank + gradient
instantiation, and every fused engine mode -- which separates Adam from the order of the gradient sum."""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import es_oracle as orc
from test_adam_parity_cpu import BETAS, EPSS, LRS, STEPS, WDS, adam_inputs, torch_adam_step

pytestmark = pytest.mark.gpu

HP = dict(lr=0.05, betas=(0.5, 0.99), eps=1e-6, weight_decay=1e-2)      # a non-default configuration


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def dev(be, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(be.device)


def host(t):
    return t.cpu().numpy()


def assert_bits(got, want, what):
    """Bit-identical fp32 arrays (NaN positions included, -0 != +0)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    bad = got.view(np.int32) != want.view(np.int32)
    bad &= ~(np.isnan(got) & np.isnan(want))
    if bad.any():
        i = np.flatnonzero(bad)[:5]
        raise AssertionError(f"{what}: {np.count_nonzero(bad)} of {bad.size} entries differ, e.g. at {i}: "
                             f"{got.reshape(-1)[i]} vs {want.reshape(-1)[i]}")


def oracle_step(theta, m, v, g, step, lr, betas, eps, wd):
    return orc.adam_step(theta, m, v, orc.negate_clamp(g), step, lr, betas[0], betas[1], eps, wd)


def grad_sums(n, P, seed):
    """Raw pair sums (the kernel divides by P): beyond +-P (the clamp), exactly onto +-1 after the division,
    one ulp either side of it, +-0 and subnormal quotients."""
    _, _, _, g = adam_inputs(n, seed)
    s = (g * np.float32(P) * np.float32(1.3)).astype(np.float32)
    fP = np.float32(P)
    special = np.array([fP, -fP, np.nextafter(fP, np.float32(np.inf)), np.nextafter(-fP, np.float32(0)),
                        np.float32(2.5) * fP, 0.0, -0.0, np.float32(1e-40) * fP, np.float32(-3e-42),
                        np.nextafter(np.float32(0), np.float32(1))], np.float32)
    k = min(n, special.size)
    s[:k] = special[:k]
    return s


def _clamp_adam(be, sums, P, theta, m, v, t, hp, with_grad=True):
    from estorch_b200.backend import adam_desc, new_state, read_state, write_state
    st = new_state(be.device)
    write_state(st, adam_step=t)
    th, mm, vv = dev(be, theta), dev(be, m), dev(be, v)
    gout = be.zeros(sums.size) if with_grad else None
    be.clamp_adam(dev(be, sums), P, th, mm, vv, st, adam_desc(**hp))
    if with_grad:
        be.clamp_adam(dev(be, sums), P, None, None, None, None, adam_desc(**hp), gout)   # clamp(-g) alone
    torch.cuda.synchronize()
    assert read_state(st)["adam_step"] == t + 1
    return host(th), host(mm), host(vv), None if gout is None else host(gout)


# ------------------------------------------------------------------ estk_clamp_adam
@pytest.mark.parametrize("betas", BETAS)
def test_clamp_adam_bit_exact_over_the_grid(be, betas):
    n, P = 4610, 96
    theta, m, v, _ = adam_inputs(n, seed=7)
    sums = grad_sums(n, P, seed=8)
    g = (sums / np.float32(P)).astype(np.float32)
    for lr in LRS:
        for eps in EPSS:
            for wd in WDS:
                for t in STEPS:
                    hp = dict(lr=lr, betas=betas, eps=eps, weight_decay=wd)
                    th, mm, vv, gp = _clamp_adam(be, sums, P, theta, m, v, t - 1, hp, with_grad=(t == 1))
                    want = oracle_step(theta, m, v, g, t, lr, betas, eps, wd)
                    what = f"lr={lr} eps={eps} wd={wd} t={t}"
                    assert_bits(mm, want[1], "m " + what)
                    assert_bits(vv, want[2], "v " + what)
                    assert_bits(th, want[0], "theta " + what)
                    if gp is not None:
                        assert_bits(gp, orc.negate_clamp(g), "clamp(-g)")


@pytest.mark.parametrize("n", [1, 7, 1001760])
def test_clamp_adam_sizes_and_grad_out(be, n):
    from estorch_b200.backend import adam_desc, new_state
    P = 64
    theta, m, v, _ = adam_inputs(n, seed=n)
    sums = grad_sums(n, P, seed=n + 1)
    g = (sums / np.float32(P)).astype(np.float32)
    st = new_state(be.device)
    th, mm, vv, gout = dev(be, theta), dev(be, m), dev(be, v), be.zeros(n)
    for t in (1, 2):                                      # the kernel advances adam_step itself
        be.clamp_adam(dev(be, sums), P, th, mm, vv, st, adam_desc(**HP), gout)
        theta, m, v = oracle_step(theta, m, v, g, t, **_hp_args(HP))
        assert_bits(host(gout), g, "grad_out")
        assert_bits(host(mm), m, f"m t={t}")
        assert_bits(host(vv), v, f"v t={t}")
        assert_bits(host(th), theta, f"theta t={t}")


def _hp_args(hp):
    return dict(lr=hp["lr"], betas=hp["betas"], eps=hp["eps"], wd=hp["weight_decay"])


# ------------------------------------------------------------------ estk_rank_grad_adam
@pytest.mark.parametrize("P,n,table", [
    (8, 1, "fp32"), (8, 7, "fp32"),
    (64, 4610, "fp32"), (64, 4610, "fp16"),               # partial sums (PS > 1)
    (64, 1001760, "fp32"), (64, 1001760, "fp16"),         # column split
    (16384, 4610, "fp32"), (16384, 1001760, "fp16"),      # P > 8192: the radix-sort instantiations
])
def test_rank_grad_adam_instantiations(be, P, n, table):
    from estorch_b200.backend import adam_desc, new_state, read_state, write_state
    rng = np.random.RandomState(P + n)
    table_len = (n + 31) // 32 * 32 + (1 << 16)
    tab = orc.round_f16(rng.standard_normal(table_len).astype(np.float32))
    tb = dev(be, tab)
    if table == "fp16":
        t16 = be.alloc(table_len, dtype=torch.float16)
        assert be.shadow_f16(tb, t16) == 0
        tb = t16
    offs = orc.noise_offsets(3, 1, 0, P // 2, table_len, n)
    order = np.argsort(offs, kind="stable").astype(np.int32)
    ret = rng.standard_normal(P).astype(np.float32)
    theta, m, v, _ = adam_inputs(n, seed=P)
    for t0, hp in ((0, HP), (999, dict(lr=0.3, betas=(0.9, 0.999), eps=0.0, weight_decay=0.5))):
        st = new_state(be.device)
        write_state(st, adam_step=t0)
        th, mm, vv, g = dev(be, theta), dev(be, m), dev(be, v), be.zeros(n)
        ranks = be.zeros(P, dtype=torch.int32)
        be.rank_grad_adam(dev(be, ret), None, 1.0, 0.0, P, tb, dev(be, offs), dev(be, order), th, mm, vv, st,
                          adam_desc(**hp), ranks, None, g)
        torch.cuda.synchronize()
        assert read_state(st)["adam_step"] == t0 + 1
        np.testing.assert_array_equal(host(ranks), orc.compute_ranks(ret))
        want = oracle_step(theta, m, v, host(g), t0 + 1, **_hp_args(hp))
        assert_bits(host(mm), want[1], f"m t={t0 + 1}")
        assert_bits(host(vv), want[2], f"v t={t0 + 1}")
        assert_bits(host(th), want[0], f"theta t={t0 + 1}")


# ------------------------------------------------------------------ torch's own Adam on the device
def _v_forms(v, g, b2):
    """The ways a CUDA build of ``v.mul_(b2).addcmul_(g, g, value=1 - b2)`` can round."""
    f = np.float32
    c, bv = f(1.0 - b2), (v * f(b2)).astype(f)
    return {"fma((1-b2)*g, g, b2*v)": orc.fma32((c * g).astype(f), g, bv),
            "fma(1-b2, g*g, b2*v)": orc.fma32(c, (g * g).astype(f), bv),
            "b2*v + ((1-b2)*g)*g": (bv + ((c * g).astype(f) * g).astype(f)).astype(f),
            "b2*v + (1-b2)*(g*g)": (bv + (c * (g * g).astype(f)).astype(f)).astype(f)}


@pytest.mark.parametrize("foreach", [False, True])
def test_torch_adam_on_the_device_witness(be, foreach, record_property, capsys):
    """A second witness: torch.optim.Adam on CUDA (weight_decay = 0), whose kernels are compiled differently
    from the CPU ones the fused step follows (the reference's arithmetic).  Which form CUDA uses is recorded,
    not forced: m must be the oracle's values (its bits, or they differ in the sign of a zero), v one of the
    known roundings of addcmul_, the same one everywhere, and theta the rest of the oracle's chain on torch's
    own m / v to within an ulp of theta and four of the update."""
    n = 1 << 16
    theta, m, v, g = adam_inputs(n, seed=5)
    gp = orc.negate_clamp(g)
    v_forms, m_forms = set(), set()
    f = np.float32
    for betas in BETAS:
        for t in (1, 10, 1000):
            got = torch_adam_step(theta, m, v, gp, t, 0.01, betas, 1e-8, 0.0, foreach=foreach, device=be.device)
            want = orc.adam_step(theta, m, v, gp, t, 0.01, betas[0], betas[1], 1e-8, 0.0)
            np.testing.assert_array_equal(got[1], want[1], err_msg=f"m betas={betas} t={t}")   # +0 == -0
            m_forms.add("the restated form" if np.array_equal(got[1].view(np.int32), want[1].view(np.int32))
                        else "the restated form up to the sign of zero")
            forms = [k for k, w in _v_forms(v, gp, betas[1]).items()
                     if np.array_equal(got[2].view(np.int32), w.view(np.int32))]
            assert forms, f"v betas={betas} t={t}: none of the known roundings"
            v_forms.add(forms[0])
            bc1, bc2 = 1.0 - betas[0] ** t, 1.0 - betas[1] ** t
            denom = ((np.sqrt(got[2]) / f(np.sqrt(bc2))).astype(f) + f(1e-8)).astype(f)
            th = (theta + ((f(-(0.01 / bc1)) * got[1]).astype(f) / denom).astype(f)).astype(f)
            upd = ((f(-(0.01 / bc1)) * got[1]).astype(f) / denom).astype(f)
            tol = np.spacing(np.abs(th)) + 4 * np.spacing(np.abs(upd))        # an ulp of theta + four of the update
            assert (np.abs(got[0] - th) <= tol).all(), f"theta betas={betas} t={t}"
    assert len(v_forms) == 1, v_forms
    record_property("torch_cuda_lerp_form", sorted(m_forms))
    record_property("torch_cuda_addcmul_form", sorted(v_forms))
    with capsys.disabled():
        print(f"\ntorch.optim.Adam(foreach={foreach}) on {be.device.type}: m is {sorted(m_forms)}, "
              f"v is {sorted(v_forms)}")


# ------------------------------------------------------------------ engine level
def _snap(es):
    from estorch_b200.backend import read_state
    return dict(grad=host(es._grad).copy(),
                slots=[(host(s.theta).copy(), host(s.m).copy(), host(s.v).copy(), read_state(s.state)["adam_step"])
                       for s in es._slots])


def check_every_step(snaps, hp):
    """Generation k moved exactly one slot's Adam step on by one, and its theta / m / v are the oracle's Adam
    of the state before and of the gradient that step consumed (ES._grad)."""
    assert len(snaps) >= 2
    for k in range(1, len(snaps)):
        before, after = snaps[k - 1], snaps[k]
        moved = [i for i, (b, a) in enumerate(zip(before["slots"], after["slots"])) if a[3] != b[3]]
        assert len(moved) == 1, moved
        i = moved[0]
        th, m, v, t = before["slots"][i]
        assert after["slots"][i][3] == t + 1
        want = oracle_step(th, m, v, after["grad"], t + 1, **_hp_args(hp))
        for got, w, what in zip(after["slots"][i][:3], want, ("theta", "m", "v")):
            assert_bits(got, w, f"{what} of slot {i}, generation {k}")
        for j, (b, a) in enumerate(zip(before["slots"], after["slots"])):
            if j != i:
                for x, y in zip(a[:3], b[:3]):
                    assert_bits(x, y, f"untouched slot {j}")


def _run(es, n_steps):
    snaps = [_snap(es)]
    es.log = lambda: snaps.append(_snap(es))
    es.train(n_steps=n_steps)
    return snaps


def _mlp_es(cls_name="ES", hp=HP, **kw):
    import estorch_b200 as E
    from test_api_cpu import MLP
    if cls_name == "ES":
        g = load_golden("es_cartpole_p64.npz")
        agent_kwargs = dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]))
        dims, P, extra = [4, 64, 64, 2], 64, {}
    else:
        g = load_golden("nsr_bipedal_p32.npz")
        agent_kwargs = dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]), bc_obs=64, bc_dim=256)
        dims, P, extra = [24, 64, 64, 4], 32, {}
    torch.manual_seed(0)
    es = getattr(E, cls_name)(MLP, E.DeviceAgent, torch.optim.Adam, population_size=P, sigma=0.05,
                              policy_kwargs={"dims": dims}, agent_kwargs=agent_kwargs, optimizer_kwargs=dict(hp),
                              noise_table_size=1 << 18, **extra, **kw)
    assert es._fused
    return es


@pytest.mark.parametrize("graph", ["1", "0"])
def test_engine_es_fused_every_step(monkeypatch, graph):
    monkeypatch.setenv("ESTORCH_B200_GRAPH", graph)
    es = _mlp_es()
    check_every_step(_run(es, 6), HP)
    graphs = sum(isinstance(v, tuple) for v in es.__dict__.get("_graphs", {}).values())
    assert (graphs >= 1) if graph == "1" else (graphs == 0)


def test_engine_nsr_es_fused_every_step():
    np.random.seed(3)
    es = _mlp_es("NSR_ES")
    check_every_step(_run(es, 4), HP)


def test_engine_conv_vbn_fused_every_step():
    import estorch_b200 as E
    from test_api_gpu import AtariPolicy
    g = torch.Generator().manual_seed(5)
    xref = torch.rand(8, 4, 84, 84, generator=g)
    obs, tgt = torch.rand(4, 4, 84, 84, generator=g), torch.randn(4, 4, generator=g)
    torch.manual_seed(1)
    es = E.ES(AtariPolicy, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.02,
              policy_kwargs=dict(n_actions=4, xref=xref), agent_kwargs=dict(obs=obs, target=tgt),
              optimizer_kwargs=dict(HP), noise_table_size=1 << 21, noise_seed=9)
    assert es._fused and es._is_conv
    check_every_step(_run(es, 2), HP)


def test_engine_mlp_population_mode_every_step():
    import estorch_b200 as E
    from _mlp_oracle import MLP
    from _pop_oracle import LinearWalker
    from test_population_cpu import DIMS
    torch.manual_seed(2)
    es = E.ES(MLP, LinearWalker, torch.optim.Adam, population_size=64, sigma=0.05,
              policy_kwargs={"dims": DIMS, "hidden": "relu", "output": "tanh"}, optimizer_kwargs=dict(HP),
              noise_table_size=1 << 18)
    assert es._population
    check_every_step(_run(es, 3), HP)


def test_mirrored_state_continues_under_torch_adam():
    """Three fused generations, the moments exposed through mirror_adam_state, then two steps of
    torch.optim.Adam (the CPU kernels: the fused step's arithmetic, see the witness above for CUDA's) on the
    same gradients give the same m / v bits as two more fused generations (weight_decay = 0: with decay, m and
    v would also inherit theta's rare one-ulp sqrt differences)."""
    hp = dict(HP, weight_decay=0.0)
    es = _mlp_es(hp=hp)
    snaps = _run(es, 5)
    fused = snaps[3:]                                    # after generations 3, 4, 5
    es2 = _mlp_es(hp=hp)
    es2.log = lambda: None
    es2.train(n_steps=3)
    slot = es2._slots[0]
    slot.mirror_adam_state()
    assert_bits(host(slot.theta), fused[0]["slots"][0][0], "theta after 3 generations")
    params = [p.detach().cpu().clone().requires_grad_(True) for p in es2.policy.parameters()]
    opt = torch.optim.Adam(params, **hp, foreach=False)
    opt.load_state_dict(es2.optimizer.state_dict())      # the mirrored moments, moved to the CPU parameters
    for k in (1, 2):
        grad = torch.from_numpy(fused[k]["grad"])
        idx = 0
        for p in params:
            p.grad = (-grad[idx: idx + p.numel()].view(p.shape)).clamp(-1.0, 1.0)
            idx += p.numel()
        opt.step()
        st = [opt.state[p] for p in params]
        m = torch.cat([s["exp_avg"].reshape(-1) for s in st])
        v = torch.cat([s["exp_avg_sq"].reshape(-1) for s in st])
        assert_bits(host(m), fused[k]["slots"][0][1], f"m, torch step {k}")
        assert_bits(host(v), fused[k]["slots"][0][2], f"v, torch step {k}")
        assert float(st[0]["step"]) == 3 + k


# ------------------------------------------------------------------ estk_rank_grad_xr_adam
def test_xr_adam_every_step_on_two_gpus(tmp_path):
    """Fused ES on two GPUs with the gradient summed over NVLink peer memory inside the rank + gradient
    kernel: every generation's step on every rank is the oracle's Adam of the summed gradient."""
    if torch.cuda.device_count() < 2:
        pytest.skip("estk_rank_grad_xr_adam needs 2 GPUs; this host has fewer, so its per-step Adam "
                    "property is checked only through estk_clamp_adam / estk_rank_grad_adam here")
    import socket
    import subprocess
    import sys
    import textwrap
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "xr_adam.py"
    script.write_text(textwrap.dedent(f"""
        import os, sys
        sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
        import test_adam_parity_gpu as T
        es = T._mlp_es()
        assert es.n_workers == 2
        snaps = T._run(es, 4)                # rank 0 alone logs; the replicas are bit-identical
        assert es.__dict__.get("_peer_ptrs") is not None, "the peer-memory reduction was not used"
        if es.rank == 0:
            T.check_every_step(snaps, T.HP)
            print("xr adam ok")
    """))
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    assert r.stdout.count("xr adam ok") == 1
