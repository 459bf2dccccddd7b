"""The oracle's Adam step (oracle/es_oracle.py ``adam_step``) against torch.optim.Adam on the CPU, bit for bit.

torch's CPU kernels round ``grad.add(param, alpha=wd)``, ``lerp_`` and ``addcmul_`` once each (fma), and
``lerp_`` switches to ``fma(w - 1, g - m, g)`` for weights |w| >= 0.5; the oracle restates those forms, and
the fused CUDA epilogue (``adam_elem``) is held bit-exact to the oracle (tests/test_adam_parity_gpu.py).
torch's CPU ``sqrt`` is not always correctly rounded, so theta is compared wherever torch's ``sqrt(v)``
equals the correctly rounded one; m and v do not depend on the square root and are compared everywhere.
Also: the fp32 fma emulation itself, the reference goldens' moments, and ``decoupled_weight_decay``."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import estorch_b200 as E
from conftest import load_golden
from _oracle_backend import OracleBackend
from oracle import es_oracle as orc

f32 = np.float32
LRS = (1e-3, 0.01, 0.3)
BETAS = ((0.9, 0.999), (0.5, 0.99), (0.3, 0.9999), (0.0, 0.999), (0.99, 0.5))
EPSS = (1e-8, 1e-3, 0.0)
WDS = (0.0, 1e-2, 0.5)
STEPS = (1, 2, 3, 10, 1000, 10 ** 5, 10 ** 6)

needs_fma = pytest.mark.skipif(torch.backends.cpu.get_cpu_capability() == "DEFAULT",
                               reason="torch's DEFAULT CPU build has no fma: not the reference's arithmetic")


# ------------------------------------------------------------------ inputs
def adam_inputs(n, seed):
    """(theta, m, v, raw estimate g) with the edges of the fused epilogue: |g| beyond the clamp, exact +-0,
    subnormals, values that round onto +-1, and m = v = 0 (0/0 = NaN with eps = 0)."""
    rng = np.random.RandomState(seed)
    theta = (rng.standard_normal(n) * 0.5).astype(f32)
    m = (rng.standard_normal(n) * 0.05).astype(f32)
    v = (rng.random(n) * 1e-2).astype(f32)
    g = (rng.standard_normal(n) * 0.7).astype(f32)
    special = np.array([3.5, -2.0, 0.0, -0.0, 1e-40, -3e-42, np.float32(1.0) + f32(2 ** -23), -1.0,
                        np.nextafter(f32(1), f32(0)), 1e-3, -7e-4, 0.25], f32)
    k = min(n, special.size)
    g[:k] = special[:k]
    if n > 2 * special.size:
        g[-k:] = special[:k]
        z = rng.choice(np.arange(special.size, n - special.size), size=max(1, n // 50), replace=False)
        m[z] = 0.0
        v[z] = 0.0
        g[z[::2]] = 0.0              # g = m = v = 0: 0/0 once eps is 0
        theta[z[1::3]] = 1e-41
    return theta, m, v, g


def torch_adam_step(theta, m, v, grad, step, lr, betas, eps, wd, foreach=False, device="cpu", **kw):
    """One torch.optim.Adam step from the given state; ``step`` counts the steps after this one."""
    p = torch.nn.Parameter(torch.from_numpy(theta.copy()).to(device))
    opt = torch.optim.Adam([p], lr=lr, betas=betas, eps=eps, weight_decay=wd, foreach=foreach, **kw)
    opt.state[p] = {"step": torch.tensor(float(step - 1)), "exp_avg": torch.from_numpy(m.copy()).to(device),
                    "exp_avg_sq": torch.from_numpy(v.copy()).to(device)}
    p.grad = torch.from_numpy(grad.copy()).to(device)
    opt.step()
    st = opt.state[p]
    return tuple(t.detach().cpu().numpy() for t in (p, st["exp_avg"], st["exp_avg_sq"]))


def torch_sqrt_exact(v):
    """Where torch's CPU sqrt(v) is the correctly rounded square root (np.sqrt is)."""
    with np.errstate(invalid="ignore"):
        return torch.from_numpy(v).sqrt().numpy().view(np.int32) == np.sqrt(v).view(np.int32)


# ------------------------------------------------------------------ fp32 fma emulation
def _round_f32(q: Fraction) -> np.float32:
    """Correctly rounded fp32 of an exact rational (nearest, ties to even), by exact comparison."""
    x = f32(float(q))
    best = None
    for c in (np.nextafter(x, f32(-np.inf)), x, np.nextafter(x, f32(np.inf))):
        if not np.isfinite(c):
            continue
        d = abs(Fraction(float(c)) - q)
        key = (d, int(np.array(c).view(np.int32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return best[1]


def test_fma32_rounds_once():
    # exact = (1 + 2^-23) + 2^-24 - 2^-70: just below an fp32 midpoint.  The fp64 sum rounds onto the
    # midpoint and a second rounding goes up; a single rounding goes down.
    a, b, c = f32(1 - 2.0 ** -23), f32((1 + 2.0 ** -23) * 2.0 ** -24), f32(1 + 2.0 ** -23)
    want = f32(1 + 2.0 ** -23)
    assert orc.fma32(a, b, c) == want
    assert f32(np.float64(a) * np.float64(b) + np.float64(c)) != want          # the double rounding
    assert orc.fma32(-a, b, -c) == -want
    rng = np.random.RandomState(3)
    a = (rng.standard_normal(3000) * np.exp2(rng.randint(-30, 30, 3000))).astype(f32)
    b = (rng.standard_normal(3000) * np.exp2(rng.randint(-30, 30, 3000))).astype(f32)
    c = (-a * b * (1 + rng.standard_normal(3000).astype(f32) * f32(2 ** -20))).astype(f32)  # cancellation
    c[::3] = (rng.standard_normal(1000) * 1e-38).astype(f32)                                 # subnormal results
    a[::7] *= f32(1e-20)
    got = orc.fma32(a, b, c)
    want = np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                     for x, y, z in zip(a, b, c)], f32)
    np.testing.assert_array_equal(got.view(np.int32), want.view(np.int32))
    assert orc.fma32(f32(0.0), f32(1.0), f32(-0.0)).view(np.int32) == 0                       # +0 + -0 = +0


# ------------------------------------------------------------------ against torch.optim.Adam
@needs_fma
@pytest.mark.parametrize("betas", BETAS)
@pytest.mark.parametrize("wd", WDS)
def test_oracle_adam_matches_torch_cpu(betas, wd):
    """Three chained steps from every starting step count, over the hyperparameter grid: each oracle step
    starts from torch's state and must give torch's m / v bits, and theta's where torch's sqrt is exact."""
    n = 4610
    th0, m0, v0, g = adam_inputs(n, seed=int(betas[0] * 100) + int(wd * 1000))
    gp = orc.negate_clamp(g)
    checked = 0
    for lr in LRS:
        for eps in EPSS:
            for t0 in STEPS:
                theta, m, v = th0, m0, v0
                for k in range(3):
                    step = t0 + k
                    g_k = gp if k == 0 else np.roll(gp, 17 * k)
                    want = torch_adam_step(theta, m, v, g_k, step, lr, betas, eps, wd)
                    got = orc.adam_step(theta, m, v, g_k, step, lr, betas[0], betas[1], eps, wd)
                    np.testing.assert_array_equal(got[1], want[1], err_msg=f"m lr={lr} eps={eps} t={step}")
                    np.testing.assert_array_equal(got[2], want[2], err_msg=f"v lr={lr} eps={eps} t={step}")
                    ok = torch_sqrt_exact(want[2])
                    assert ok.mean() > 0.9
                    np.testing.assert_array_equal(got[0][ok], want[0][ok], err_msg=f"theta lr={lr} eps={eps} t={step}")
                    if eps == 0.0 and wd == 0.0:
                        assert np.isnan(want[0]).any()               # the 0/0 entries are in the vector
                    theta, m, v = want
                    checked += 1
    assert checked == len(LRS) * len(EPSS) * len(STEPS) * 3


@needs_fma
@pytest.mark.parametrize("n", [1, 7, 33])
def test_oracle_adam_matches_torch_cpu_short_vectors(n):
    """Vectors shorter than one SIMD register: torch's scalar loop rounds the same way."""
    theta, m, v, g = adam_inputs(n, seed=n)
    gp = orc.negate_clamp(g)
    for betas in BETAS:
        for wd in WDS:
            want = torch_adam_step(theta, m, v, gp, 2, 0.01, betas, 1e-8, wd)
            got = orc.adam_step(theta, m, v, gp, 2, 0.01, betas[0], betas[1], 1e-8, wd)
            np.testing.assert_array_equal(got[1], want[1])
            np.testing.assert_array_equal(got[2], want[2])
            ok = torch_sqrt_exact(want[2])
            np.testing.assert_array_equal(got[0][ok], want[0][ok])


def test_lerp_branch_at_small_beta1():
    """beta1 <= 0.5 takes torch's large-weight lerp: beta1 = 0 gives m = g exactly (the small-weight form
    m + 1 * (g - m) rounds)."""
    rng = np.random.RandomState(1)
    m = (rng.standard_normal(4096) * 0.3).astype(f32)
    g = (rng.standard_normal(4096) * 0.3).astype(f32)
    z = np.zeros(4096, f32)
    _, m1, _ = orc.adam_step(z, m, z, g, 1, beta1=0.0)
    np.testing.assert_array_equal(m1, g)
    assert np.count_nonzero((m + (g - m)).astype(f32) != g) > 0


# ------------------------------------------------------------------ the reference goldens
GOLDENS_WITH_MOMENTS = ["es_tiny_p8", "es_cartpole_p64", "es_tanh_cartpole_p64", "es_elu_cartpole_p64",
                        "es_xent_p64", "es_leaky_xent_p64", "es_pop_walker_p64"]


@pytest.mark.parametrize("name", GOLDENS_WITH_MOMENTS)
def test_oracle_adam_chain_reproduces_golden_moments(name):
    """The unmodified reference's Adam moments after its generations, bit for bit; its theta after each
    step wherever its sqrt was the correctly rounded one."""
    g = load_golden(f"{name}.npz")
    n = g["theta0"].size
    m, v = np.zeros(n, f32), np.zeros(n, f32)
    for gen in range(len(g["grad"])):
        th, m, v = orc.adam_step(g["theta_before"][gen], m, v, orc.negate_clamp(g["grad"][gen]), gen + 1, lr=0.01)
        ok = torch_sqrt_exact(v)
        np.testing.assert_array_equal(th[ok], g["theta_after"][gen][ok])
    np.testing.assert_array_equal(m, g["m_final"])
    np.testing.assert_array_equal(v, g["v_final"])


# ------------------------------------------------------------------ decoupled weight decay
class _MLP(torch.nn.Module):
    def __init__(self, dims):
        super().__init__()
        self.net = torch.nn.Sequential(torch.nn.Linear(dims[0], dims[1]), torch.nn.ReLU(),
                                       torch.nn.Linear(dims[1], dims[2]))

    def forward(self, x):
        return self.net(x)


def _es(optimizer_kwargs):
    g = load_golden("es_cartpole_p64.npz")

    class Rec(E.ES):
        def log(self):
            self.rec.append((torch.cat([p.grad.reshape(-1) for p in self.policy.parameters()]).clone(),
                             torch.nn.utils.parameters_to_vector(self.policy.parameters()).detach().clone()))
    es = Rec(_MLP, E.DeviceAgent, torch.optim.Adam, population_size=16, sigma=0.1, policy_kwargs={"dims": [4, 32, 2]},
             agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"])),
             optimizer_kwargs=optimizer_kwargs, noise_table_size=1 << 14, _backend=OracleBackend())
    es.rec = []
    return es


def test_decoupled_weight_decay_selects_hooks_mode():
    """torch's ``decoupled_weight_decay=True`` is AdamW's theta *= 1 - lr * wd: the fused epilogue's L2 decay
    through the moments is a different optimizer, so hooks mode (torch's own step) serves it."""
    kw = {"lr": 0.05, "weight_decay": 0.1}
    assert _es(kw)._fused
    es = _es(dict(kw, decoupled_weight_decay=True))
    assert not es._fused
    theta0 = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().clone()
    es.train(n_steps=3)
    # theta after every generation is torch's AdamW-style step of the gradient that generation consumed
    p = torch.nn.Parameter(theta0.clone())
    opt = torch.optim.Adam([p], **kw, decoupled_weight_decay=True, foreach=False)
    l2 = (theta0.numpy(), np.zeros_like(theta0.numpy()), np.zeros_like(theta0.numpy()))
    for step, (grad, theta) in enumerate(es.rec, 1):
        p.grad = grad.clone()
        opt.step()
        np.testing.assert_array_equal(theta.numpy(), p.detach().numpy())
        l2 = orc.adam_step(*l2, grad.numpy(), step, lr=0.05, weight_decay=0.1)
    assert not np.array_equal(l2[0], es.rec[-1][1].numpy())         # L2 decay would have moved theta elsewhere


@pytest.mark.parametrize("flag", ["decoupled_weight_decay", "amsgrad", "maximize"])
def test_fused_step_refuses_flags_switched_on_later(flag):
    es = _es({"lr": 0.05, "weight_decay": 0.1})
    es.log = lambda: None                   # fused mode leaves .grad unset
    assert es._fused
    es.train(n_steps=1)
    es.optimizer.param_groups[0][flag] = True
    with pytest.raises(ValueError, match=flag):
        es.train(n_steps=1)
