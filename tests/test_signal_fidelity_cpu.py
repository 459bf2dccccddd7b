"""The float64 reference of an evaluate call (tests/_fp64_signal.py) against an independent torch.float64
forward, its error bound against the fp32 restatements of every back end, and the rounding models of the
tensor-core modes measured on what ES consumes: pair differences, ranks and the gradient, across sigma and
the weight scale.  No GPU: the kernels themselves are measured the same way in test_signal_fidelity_gpu.py."""
import numpy as np
import pytest
import torch

from estorch_b200.estorch import AUTO_F16_MIN_SIGMA
from oracle import es_oracle as orc
import _mlp_oracle as mlp
import _fp64_signal as sig


def init_theta(dims, scale, seed=0):
    """nn.Linear's initialisation of an MLP, times ``scale``: the weights grown by training."""
    torch.manual_seed(seed)
    mods = [torch.nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])]
    flat = torch.cat([t.detach().reshape(-1) for m in mods for t in (m.weight, m.bias)]).numpy()
    return (flat * np.float32(scale)).astype(np.float32)


def noise(n, pairs, seed=5):
    table = orc.philox_normal_table((n + 31) // 32 * 32 + 32 * 8 * pairs, seed)
    return table, orc.noise_offsets(seed, 0, 0, pairs, table.size, n)


def task(dims, B, loss, obs_scale=1.0, seed=1):
    rng = np.random.RandomState(seed)
    obs = (rng.standard_normal((B, dims[0])) * obs_scale).astype(np.float32)
    if loss == "xent":
        return obs, np.eye(dims[-1], dtype=np.float32)[rng.randint(0, dims[-1], B)]
    return obs, rng.standard_normal((B, dims[-1])).astype(np.float32)


# ------------------------------------------------------------------ the helper against torch.float64
@pytest.mark.parametrize("hidden", sorted(mlp.HIDDEN_CODES))
@pytest.mark.parametrize("output,loss", [("identity", "mse"), ("tanh", "mse"), ("identity", "xent")])
def test_reference_matches_torch_float64_sequential(hidden, output, loss):
    dims, B, pairs, sigma = [7, 33, 17, 5], 9, 4, 0.05
    theta = init_theta(dims, 3.0)
    table, offs = noise(theta.size, pairs)
    obs, tgt = task(dims, B, loss)
    if loss == "xent":
        tgt = np.random.RandomState(2).rand(B, dims[-1]).astype(np.float32)      # soft targets
    rows = sig.members(theta, table, offs, sigma)
    perturbed, _ = orc.sample_population(theta, table, offs, sigma)
    np.testing.assert_array_equal(rows, perturbed)
    # the rows are what perturb_rows forms: eps = fp32(sigma * T), W = fp32(theta +- eps)
    eps = (np.float32(sigma) * table[offs[1]: offs[1] + theta.size]).astype(np.float32)
    np.testing.assert_array_equal(rows[pairs + 1], (theta - eps).astype(np.float32))
    r64, tau = sig.mlp_reference(rows, dims, obs, tgt, hidden, output, loss)
    net = mlp.MLP(dims, hidden, output).double()
    t = torch.from_numpy(tgt).double()
    want = []
    for row in rows:
        torch.nn.utils.vector_to_parameters(torch.from_numpy(row.astype(np.float64)), net.parameters())
        with torch.no_grad():
            y = net(torch.from_numpy(obs).double())
        if loss == "xent":
            want.append(float((t * torch.log_softmax(y, -1)).sum(-1).mean()))
        else:
            want.append(float(-((y - t) ** 2).mean()))
    np.testing.assert_allclose(r64, want, rtol=1e-12, atol=0)
    # the bound covers the fp32 forward, and is not vacuous: within 10^4 ulps of the return
    r32, _ = mlp.evaluate_population(rows, dims, obs, tgt, mlp.code(hidden, output, loss))
    assert np.all(np.abs(r32 - r64) <= tau)
    assert np.all(tau < 1e4 * sig.U32 * np.abs(r64))


def test_metrics_of_known_perturbations():
    r64 = np.array([1.0, 2.0, 3.0, 4.0, 1.5, 2.5, 2.0, 4.5])
    same = sig.signal_metrics(r64, r64)
    assert same["returns_max_rel"] == same["diff_max_over_std"] == same["diff_wrong_sign"] == 0
    assert same["rank_max_disp"] == 0
    r = r64.copy()
    r[2] = 1.9                    # member 2 drops below members 1, 6 and 5: D_2 = 3.0 - 2.0 -> -0.1
    m = sig.signal_metrics(r, r64)
    assert m["diff_wrong_sign"] == 0.25 and m["rank_max_disp"] == 3
    assert m["diff_max_over_std"] == pytest.approx(1.1 / np.std(r64[:4] - r64[4:]))
    tau = np.full(8, 0.05)
    viol, pinned = sig.rank_violations(r, r64, tau)
    # 1 and 6 tie at 2.0 in float64 and are excused; 2 and 5 have no neighbour within 0.1 and moved
    assert list(viol) == [2, 5] and pinned == 6
    viol, pinned = sig.rank_violations(r, r64, np.full(8, 0.6))
    assert viol.size == 0 and pinned == 0


# ------------------------------------------------------------------ fp32 restatements keep exact ranks
def _check_fp32(r32, r64, tau):
    assert np.all(np.abs(np.asarray(r32, np.float64) - r64) <= tau)
    viol, pinned = sig.rank_violations(r32, r64, tau)
    assert viol.size == 0
    return pinned


@pytest.mark.parametrize("scale", [1.0, 8.0])
def test_fp32_restatements_keep_exact_ranks(scale):
    """The fp32 oracles of the MLP, recurrent and convolutional back ends keep every member's float64 rank
    wherever no float64 neighbour lies within the bound: the bound the GPU test holds the kernels to."""
    import _cnn_oracle as cnn
    import _rnn_oracle as rnn
    import _seq_oracle as seq
    pairs, sigma = 16, 0.02
    pinned = {}
    dims = [16, 64, 64, 4]
    theta = init_theta(dims, scale)
    table, offs = noise(theta.size, pairs)
    obs, tgt = task(dims, 64, "mse")
    rows = sig.members(theta, table, offs, sigma)
    r32, _ = mlp.evaluate_population(rows, dims, obs, tgt)
    pinned["mlp"] = _check_fp32(r32, *sig.mlp_reference(rows, dims, obs, tgt))
    gdims = (5, 32, 3)
    g = np.random.RandomState(3)
    gtheta = ((g.rand(rnn.param_count("gru", gdims)) * 2 - 1) / np.sqrt(32) * scale).astype(np.float32)
    table, offs = noise(gtheta.size, pairs)
    gobs = g.standard_normal((8, 6, 5)).astype(np.float32)
    gtgt = (g.rand(8, 6, 3) * 1.6 - 0.8).astype(np.float32)
    rows = sig.members(gtheta, table, offs, sigma)
    r32 = seq.seq_returns32(seq.seq_outputs32(rows, "gru", list(gdims), gobs, False), gtgt, False)
    pinned["gru"] = _check_fp32(r32, *sig.seq_reference(rows, "gru", list(gdims), gobs, gtgt))
    cdims, code = cnn.pack((1, 12, 12), [(8, 3, 2, 1)], [16, 4]), 1 << 24
    ctheta = (g.uniform(-1, 1, cnn.param_count(cdims, 1)) / 3 * scale).astype(np.float32)
    table, offs = noise(ctheta.size, pairs)
    cobs, ctgt = g.standard_normal((8, 1, 12, 12)).astype(np.float32), g.standard_normal((8, 4)).astype(np.float32)
    rows = sig.members(ctheta, table, offs, sigma)
    r32 = cnn.returns_of(np.stack([cnn.forward(r, cdims, code, cobs) for r in rows]), ctgt, False)
    pinned["cnn"] = _check_fp32(r32, *sig.cnn_reference(rows, cdims, code, cobs, ctgt))
    # the bar binds: at sigma = 0.02 most members have no float64 neighbour within the bound
    assert all(p >= pairs for p in pinned.values()), pinned


# ------------------------------------------------------------------ the rounding models, measured
SWEEP_DIMS, SWEEP_B, SWEEP_PAIRS = [64, 256, 256, 32], 256, 32


@pytest.fixture(scope="module")
def sweep():
    """Signal metrics of the fp32, f16 and bf16 rounding models on the ReLU [64, 256, 256, 32] squared-error
    task (B = 256, 32 pairs), per (weight scale, sigma)."""
    n = orc.mlp_param_count(SWEEP_DIMS)
    table, offs = noise(n, SWEEP_PAIRS)
    obs, tgt = task(SWEEP_DIMS, SWEEP_B, "mse")
    out = {}
    for scale in (1.0, 4.0, 8.0):
        theta = init_theta(SWEEP_DIMS, scale)
        for sigma in (0.02, 5e-3, 1e-3, 2e-4):
            rows = sig.members(theta, table, offs, sigma)
            r64, tau = sig.mlp_reference(rows, SWEEP_DIMS, obs, tgt)
            g64 = sig.gradient64(r64, table, offs, n)
            for mode in ("fp32", "f16", "bf16"):
                r, _ = mlp.evaluate_population(rows, SWEEP_DIMS, obs, tgt, precision=mode)
                m = sig.signal_metrics(r, r64, sig.gradient64(r, table, offs, n), g64)
                m["rank_violations"] = int(sig.rank_violations(r, r64, tau)[0].size)
                out[mode, scale, sigma] = m
    return out


def test_emulated_fp32_keeps_the_float64_ranks(sweep):
    """fp32 reorders only members whose float64 returns lie within the bound of each other: a swap of
    two near-ties at most, and then the gradient moves by that one swap."""
    for (mode, scale, sigma), m in sweep.items():
        if mode == "fp32":
            assert m["rank_violations"] == 0 and m["rank_max_disp"] <= 1, (scale, sigma, m)
            assert m["grad_rel_l2"] < 1e-2, (scale, sigma, m)


def test_emulated_f16_within_the_documented_domain(sweep):
    """The domain ES documents for "f16" (measured on an H100, test_signal_fidelity_gpu.py): gradient rel-L2
    <= 3e-2 against float64 at sigma >= AUTO_F16_MIN_SIGMA with weights up to 8x their initialisation.
    Below it f16 misses that bar at grown weights (so ``eval_precision="auto"`` picks fp32 there), and at
    sigma = 2e-4 f16 and bf16 reorder members whose float64 returns are far apart."""
    for (mode, scale, sigma), m in sweep.items():
        if mode == "f16" and sigma >= AUTO_F16_MIN_SIGMA:
            assert m["grad_rel_l2"] <= 3e-2, (scale, sigma, m)
    assert max(sweep["f16", s, 1e-3]["grad_rel_l2"] for s in (1.0, 4.0)) > 3e-2
    assert min(sweep["f16", s, 2e-4]["grad_rel_l2"] for s in (4.0, 8.0)) > 3e-2
    # bf16's 8-bit significand is the larger error below the domain
    for sigma in (1e-3, 2e-4):
        for scale in (1.0, 4.0, 8.0):
            assert sweep["bf16", scale, sigma]["grad_rel_l2"] > sweep["f16", scale, sigma]["grad_rel_l2"]
    # the returns alone do not show it: f16 stays within 2e-4 (max-norm relative) in every cell
    assert max(m["returns_max_rel"] for (mode, *_), m in sweep.items() if mode == "f16") < 2e-4


@pytest.mark.parametrize("sigma,want", [(AUTO_F16_MIN_SIGMA, "f16"), (0.05, "f16"),
                                        (np.nextafter(AUTO_F16_MIN_SIGMA, 0), "fp32"), (1e-3, "fp32")])
def test_auto_picks_fp32_below_the_sigma_threshold(sigma, want):
    """``eval_precision="auto"`` on a shape the f16 kernel accepts: "f16" from AUTO_F16_MIN_SIGMA up, "fp32"
    below it; an explicit "f16" is honoured at any sigma."""
    from estorch_b200 import ES, DeviceAgent
    from _mlp_oracle import MLP
    from _oracle_backend import OracleBackend
    dims = [64, 256, 64]
    g = torch.Generator().manual_seed(0)
    obs, tgt = torch.randn(256, 64, generator=g), torch.randn(256, 64, generator=g)

    def make(precision):
        return ES(MLP, DeviceAgent, torch.optim.Adam, population_size=8, sigma=float(sigma),
                  policy_kwargs={"dims": dims, "hidden": "relu"}, agent_kwargs={"obs": obs, "target": tgt},
                  noise_table_size=1 << 16, eval_precision=precision,
                  _backend=OracleBackend(tensor_core=True))
    assert make("auto")._precision == want
    assert make("f16")._precision == "f16"
