"""The public API on a real H100, through the C ABI (no stand-in): parity with the
reference-generated goldens and with the oracle."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import es_oracle as orc
import estorch_b200 as E
from test_api_cpu import MLP, HostAgent

pytestmark = pytest.mark.gpu


def _set_theta(es, module, flat):
    with torch.no_grad():
        idx = 0
        for p in module.parameters():
            p.data.copy_(torch.from_numpy(flat[idx: idx + p.numel()]).view(p.shape))
            idx += p.numel()


def test_smoke_entry():
    import __graft_entry__
    __graft_entry__.smoke()


def test_es_fused_three_generations_vs_reference_golden():
    g = load_golden("es_cartpole_p64.npz")
    rec = []

    class R(E.ES):
        def log(self):
            rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward,
                            best=self.best_reward, ranks=self._ranks.cpu().numpy().copy(),
                            grad=self._grad.cpu().numpy().copy(),
                            theta=self._slots[0].theta.cpu().numpy().copy()))
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.1,
           policy_kwargs={"dims": [4, 64, 64, 2]},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"])),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]))
    assert es._fused and es._be.name == "cuda" and next(es.policy.parameters()).is_cuda
    es._table.copy_(torch.from_numpy(g["table"]))
    _set_theta(es, es.policy, g["theta0"])
    es.train(n_steps=3)
    n = 4610
    theta, m, v = g["theta0"].copy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
    for gen in range(3):
        r = rec[gen]
        # stage A: returns of the fp32 evaluate kernel vs the oracle on the SAME theta
        offs = g["offsets"][gen]
        pop, eps = orc.sample_population(theta, g["table"], offs, 0.1)
        want, _ = orc.evaluate_population(pop, [4, 64, 64, 2], g["obs"], g["target"])
        assert rel_err(r["returns"][:, 0], want) < 5e-6
        # stage B: on the GPU's own return bits -> bit-exact ranks, grad/theta within 1e-5
        ret = r["returns"][:, 0]
        np.testing.assert_array_equal(r["ranks"], orc.compute_ranks(ret))
        grad = orc.calculate_grad(ret, eps, 0.1)
        assert rel_err(r["grad"], grad) < 1e-5
        th, m, v = orc.adam_step(theta, m, v, orc.negate_clamp(r["grad"]), gen + 1)
        assert rel_err(r["theta"], th) < 1e-6
        assert abs(r["episode"] - float(orc.synthetic_return(orc.mlp_forward(th, [4, 64, 64, 2], g["obs"]),
                                                             g["target"]))) < 1e-5
        theta = r["theta"]
        # and the whole trajectory stays on the reference's (1e-4: chained Adam steps)
        assert rel_err(r["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-4
    assert rec[2]["best"] == pytest.approx(float(g["best_reward"][2]), abs=1e-4)
    st = es.optimizer.state[next(es.policy.parameters())]
    assert float(st["step"]) == 3.0 and st["exp_avg"].is_cuda


def test_host_agent_path_on_gpu_rows():
    g = load_golden("es_cartpole_p64.npz")
    rec = []

    class R(E.ES):
        def log(self):
            rec.append(self.population_returns.copy())
    es = R(MLP, HostAgent, torch.optim.Adam, population_size=64, sigma=0.1,
           policy_kwargs={"dims": [4, 64, 64, 2]},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"])),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]))
    assert not es._fused and not next(es.policy.parameters()).is_cuda   # policy stays on `device` (cpu)
    es._table.copy_(torch.from_numpy(g["table"]))
    torch.nn.utils.vector_to_parameters(torch.from_numpy(g["theta0"].copy()), es.policy.parameters())
    es.train(n_steps=2)
    for gen in range(2):
        assert rel_err(rec[gen][:, 0], g["returns"][gen][:, 0]) < 1e-5
    theta = torch.nn.utils.parameters_to_vector(es.policy.parameters()).detach().numpy()
    assert rel_err(theta, g["theta_after"][1]) < 1e-4


@pytest.mark.parametrize("algo,cls", [("ns", "NS_ES"), ("nsr", "NSR_ES"), ("nsra", "NSRA_ES")])
def test_ns_family_fused_vs_reference_golden(algo, cls):
    g = load_golden(f"{algo}_bipedal_p32.npz")
    kw = {"weight_t": 2} if algo == "nsra" else {}
    rec = []

    class R(getattr(E, cls)):
        def log(self):
            rec.append(dict(returns=self.population_returns.copy(), episode=self.episode_reward, idx=self.idx,
                            weight=getattr(self, "weight", None)))
    np.random.seed(123)
    es = R(MLP, E.DeviceAgent, torch.optim.Adam, population_size=32, sigma=0.02,
           policy_kwargs={"dims": [24, 64, 64, 4]},
           agent_kwargs=dict(obs=torch.from_numpy(g["obs"]), target=torch.from_numpy(g["target"]),
                             bc_obs=64, bc_dim=256),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=len(g["table"]), noise_seed=int(g["noise_seed"]), **kw)
    assert es._fused
    es._table.copy_(torch.from_numpy(g["table"]))
    for i, (p, _) in enumerate(es.meta_population):
        _set_theta(es, p, g["meta_theta0"][i])
    es._archive = [a.copy() for a in g["archive0"]]
    np.random.seed(123)
    es.train(n_steps=len(g["grad"]))
    for gen in range(len(g["grad"])):
        assert rec[gen]["idx"] == int(g["idx"][gen])
        assert rel_err(rec[gen]["returns"][:, 0], g["returns"][gen][:, 0]) < 1e-4
        assert rel_err(rec[gen]["returns"][:, 1], g["returns"][gen][:, 1]) < 1e-4
        assert abs(rec[gen]["episode"] - float(g["episode_reward"][gen])) < 1e-4
        if algo == "nsra":
            assert rec[gen]["weight"] == pytest.approx(float(g["weight"][gen]))
    final = np.stack([p_.detach().cpu().numpy() for p_ in
                      [torch.nn.utils.parameters_to_vector(p.parameters()) for p, _ in es.meta_population]])
    assert rel_err(final, g["meta_theta_final"]) < 5e-3


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("auto", 1e-5), ("bf16", 1e-3), ("bf16s", 1e-3)])
def test_north_star_shape_one_generation_properties(precision, tol):
    """BASELINE north-star sizes (P=4096, n=1,001,760, B=256): one fused generation;
    ranks are a permutation, theta moved by ~lr everywhere, returns finite/unique."""
    dims = [128, 512, 512, 512, 512, 288]
    g = torch.Generator().manual_seed(1234)
    obs, tgt = torch.randn(256, 128, generator=g), torch.randn(256, 288, generator=g)

    class Q(E.ES):
        def log(self):
            pass
    torch.manual_seed(0)
    es = Q(MLP, E.DeviceAgent, torch.optim.Adam, population_size=4096, sigma=0.02,
           policy_kwargs={"dims": dims}, agent_kwargs=dict(obs=obs, target=tgt),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 26, eval_precision=precision)
    assert es.n_parameters == 1001760 and es._fused and es._precision == ("f16" if precision == "auto" else precision)
    before = es._slots[0].theta.clone()
    es.train(n_steps=1)
    ret = es.population_returns[:, 0]
    # (fp32 returns DO tie at this scale -- ~30k representable values around -1.0 for
    #  4096 members -- so the stable-by-index tie rule is exercised here)
    assert np.isfinite(ret).all() and len(np.unique(ret)) > 2048
    ranks = es._ranks.cpu().numpy()
    np.testing.assert_array_equal(np.sort(ranks), np.arange(4096))
    np.testing.assert_array_equal(ranks, orc.compute_ranks(ret))
    moved = (es._slots[0].theta - before).abs()
    gr = es._grad.abs()
    ok = gr > 1e-2 * gr.max()
    assert float((moved[ok] - 0.01).abs().max()) < 1e-5
    # spot-check 3 members' returns against the oracle forward on materialised rows
    pop = es.population_parameters
    for member in (0, 2047, 4095):
        row = pop[member].cpu().numpy()
        want = orc.synthetic_return(orc.mlp_forward(row, dims, obs.numpy()), tgt.numpy())
        assert abs(ret[member] - float(want)) < tol * abs(float(want))


class AtariPolicy(torch.nn.Module):
    """Architecture of the reference's examples/atari.py:14-37, built with estorch_b200's VirtualBatchNorm."""
    def __init__(self, n_actions, xref):
        super().__init__()
        self.xref = xref
        self.conv1 = torch.nn.Conv2d(4, 16, 8, 4)
        self.bn1 = E.VirtualBatchNorm(16)
        self.conv2 = torch.nn.Conv2d(16, 32, 4, 2)
        self.bn2 = E.VirtualBatchNorm(32)
        self.fc1 = torch.nn.Linear(2592, 256)
        self.fc2 = torch.nn.Linear(256, n_actions)

    def forward(self, x):
        F = torch.nn.functional
        xref = F.relu(self.bn1(self.conv1(self.xref.to(x.device))))
        xref = F.relu(self.bn2(self.conv2(xref)))
        x = F.relu(self.bn1(self.conv1(x)))
        x = F.relu(self.bn2(self.conv2(x)))
        return self.fc2(F.relu(self.fc1(x.view(-1, 2592))))


def test_conv_vbn_policy_fused_generation_vs_oracle():
    """BASELINE config 5 shape (Atari conv + VirtualBatchNorm), small sizes: one fused generation;
    returns vs the oracle's atari_forward, ranks / gradient / Adam vs the oracle on the same return bits."""
    g = torch.Generator().manual_seed(5)
    xref = torch.rand(8, 4, 84, 84, generator=g)
    obs, tgt = torch.rand(4, 4, 84, 84, generator=g), torch.randn(4, 4, generator=g)
    rec = {}

    class Q(E.ES):
        def log(self):
            rec["returns"] = self.population_returns[:, 0].copy()
            rec["episode"] = self.episode_reward
    torch.manual_seed(1)
    P, sigma, table_len, seed = 8, 0.02, 1 << 21, 9
    es = Q(AtariPolicy, E.DeviceAgent, torch.optim.Adam, population_size=P, sigma=sigma,
           policy_kwargs=dict(n_actions=4, xref=xref), agent_kwargs=dict(obs=obs, target=tgt),
           optimizer_kwargs={"lr": 0.01}, noise_table_size=table_len, noise_seed=seed)
    assert es._fused and es._is_conv and es.n_parameters == 677268
    theta0 = es._slots[0].theta.cpu().numpy().copy()
    table = es._table.cpu().numpy()
    es.train(n_steps=1)
    n = theta0.size
    offs = orc.noise_offsets(seed, 0, 0, P // 2, table_len, n)
    pop, eps = orc.sample_population(theta0, table, offs, sigma)
    want = np.array([orc.synthetic_return(orc.atari_forward(pop[i], 4, xref.numpy(), obs.numpy()), tgt.numpy())
                     for i in range(P)])
    assert rel_err(rec["returns"], want) < 5e-5
    np.testing.assert_array_equal(es._ranks.cpu().numpy(), orc.compute_ranks(rec["returns"]))
    grad = orc.calculate_grad(rec["returns"], eps, sigma)
    assert rel_err(es._grad.cpu().numpy(), grad) < 1e-5
    th, _, _ = orc.adam_step(theta0, np.zeros(n, np.float32), np.zeros(n, np.float32),
                             orc.negate_clamp(es._grad.cpu().numpy()), 1)
    assert rel_err(es._slots[0].theta.cpu().numpy(), th) < 1e-6
    ep = float(orc.synthetic_return(orc.atari_forward(th, 4, xref.numpy(), obs.numpy()), tgt.numpy()))
    assert abs(rec["episode"] - ep) < 5e-5 * abs(ep)
    # the torch module (parameters are views of the flat device theta) agrees with the kernel
    # (cuDNN convolutions run in TF32 by default, hence the loose 1e-3)
    with torch.no_grad():
        out = es.policy(obs.to(es._dev))
    assert abs(float(-((out - tgt.to(es._dev)) ** 2).mean()) - rec["episode"]) < 1e-3 * abs(ep)


def test_deferred_post_update_rollout_is_equivalent():
    """With log_interval > 1 the post-update rollout of a generation is folded into the next
    generation's evaluate launch; everything observable must be identical to log_interval = 1."""
    dims = [128, 512, 288]
    g = torch.Generator().manual_seed(2)
    obs, tgt = torch.randn(256, 128, generator=g), torch.randn(256, 288, generator=g)
    out = {}
    for li in (1, 3):
        seen = []

        class Q(E.ES):
            def log(self):
                seen.append((self.step, self.episode_reward, self.best_reward))
        torch.manual_seed(4)
        es = Q(MLP, E.DeviceAgent, torch.optim.Adam, population_size=128, sigma=0.02, policy_kwargs={"dims": dims},
               agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 22,
               log_interval=li)
        assert es._precision == "f16"
        es.train(n_steps=7)
        out[li] = dict(theta=es._slots[0].theta.clone(), best=es._slots[0].best_theta.clone(), seen=seen,
                       ep=es.episode_reward, br=es.best_reward, ret=es.population_returns.copy())
    a, b = out[1], out[3]
    assert torch.equal(a["theta"], b["theta"]) and torch.equal(a["best"], b["best"])
    assert a["ep"] == b["ep"] and a["br"] == b["br"]
    np.testing.assert_array_equal(a["ret"], b["ret"])
    assert [s for s, _, _ in b["seen"]] == [2, 5] and len(a["seen"]) == 7
    for step, ep, br in b["seen"]:                     # the logged generations report the same values
        assert (step, ep, br) == a["seen"][step]


# ------------------------------------------------------------------ checkpoint / resume and the launcher, on the device
@pytest.mark.parametrize("precision", ["fp32", "auto"])
def test_checkpoint_resume_is_bit_identical_on_device(tmp_path, precision):
    """save_checkpoint() after 2 generations, 2 more; a fresh instance that loads the checkpoint and
    runs 2 generations ends with bit-identical theta / Adam moments / best snapshot (the noise table is
    regenerated from the seed, the generation counter and the Adam step live in estk_state)."""
    dims = [128, 512, 288] if precision == "auto" else [4, 64, 64, 2]
    g = torch.Generator().manual_seed(9)
    obs, tgt = torch.randn(256, dims[0], generator=g), torch.randn(256, dims[-1], generator=g)

    def make():
        torch.manual_seed(3)
        es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.05, policy_kwargs={"dims": dims},
                  agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 20,
                  eval_precision=precision, log_interval=2)
        es.log = lambda: None
        return es
    a = make()
    a.train(n_steps=2)
    path = str(tmp_path / "ck.pt")
    a.save_checkpoint(path)
    a.train(n_steps=3)
    b = make()
    b.load_checkpoint(path)
    assert b._generation == 2
    b.train(n_steps=3)
    sa, sb = a._slots[0], b._slots[0]
    for x, y in ((sa.theta, sb.theta), (sa.m, sb.m), (sa.v, sb.v), (sa.best_theta, sb.best_theta)):
        assert torch.equal(x, y)
    assert a.best_reward == b.best_reward and a.episode_reward == b.episode_reward and a._generation == b._generation == 5
    np.testing.assert_array_equal(a.population_returns, b.population_returns)


def test_graph_replay_equals_eager(monkeypatch):
    """A generation replayed from a CUDA graph (the default after the first sighting of a configuration)
    leaves exactly the state the eager launches leave."""
    dims = [128, 512, 288]
    g = torch.Generator().manual_seed(2)
    obs, tgt = torch.randn(256, 128, generator=g), torch.randn(256, 288, generator=g)
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ESTORCH_B200_GRAPH", mode)
        torch.manual_seed(4)
        es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=128, sigma=0.02, policy_kwargs={"dims": dims},
                  agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 22,
                  log_interval=4)
        es.log = lambda: None
        es.train(n_steps=13)
        out[mode] = (es._slots[0].theta.clone(), es._slots[0].best_theta.clone(), es.episode_reward, es.best_reward,
                     es.population_returns.copy(), sum(isinstance(v, tuple) for v in es.__dict__.get("_graphs", {}).values()))
    a, b = out["1"], out["0"]
    assert a[5] >= 1 and b[5] == 0                       # graphs were actually used / not used
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3]
    np.testing.assert_array_equal(a[4], b[4])


def test_train_n_proc_2_reexecs_under_torchrun(tmp_path):
    """train(n_proc=2) in a plain `python script.py` re-executes the script under torch.distributed.run with
    one process per GPU, like the reference's _fork under mpirun (estorch.py:41-56, :305); both ranks end with
    the same parameters and rank 0 alone logs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess, sys, os, textwrap
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "user_script.py"
    script.write_text(textwrap.dedent(f"""
        import os, sys, numpy as np, torch
        sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
        import estorch_b200 as E
        from test_api_cpu import MLP
        g = torch.Generator().manual_seed(1)
        obs, tgt = torch.randn(256, 128, generator=g), torch.randn(256, 288, generator=g)
        class Q(E.ES):
            def log(self):
                open(os.path.join({str(tmp_path)!r}, f"log_rank{{self.rank}}.txt"), "a").write(f"{{self.step}}\\n")
        es = Q(MLP, E.DeviceAgent, torch.optim.Adam, population_size=256, sigma=0.02, policy_kwargs={{"dims": [128, 512, 288]}},
               agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={{"lr": 0.01}}, noise_table_size=1 << 22)
        es.train(n_steps=3, n_proc=2)
        torch.cuda.synchronize()
        np.save(os.path.join({str(tmp_path)!r}, f"theta_rank{{es.rank}}.npy"), es._slots[0].theta.cpu().numpy())
    """))
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    t0, t1 = np.load(tmp_path / "theta_rank0.npy"), np.load(tmp_path / "theta_rank1.npy")
    np.testing.assert_array_equal(t0, t1)
    assert (tmp_path / "log_rank0.txt").read_text().split() == ["0", "1", "2"] and not (tmp_path / "log_rank1.txt").exists()


def test_peer_memory_gradient_sum_matches_nccl_on_2_gpus():
    """tools/multi_gpu_check.py under torchrun on 2 GPUs: fused ES and NSRA-ES with the gradient summed inside the
    kernel over NVLink peer memory (estk_rank_grad_xr_adam) and with NCCL -- replicas bit-identical across
    ranks, CUDA-graph replay == eager launches, the two reductions equal up to the order of an fp32 sum."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess, sys, os, socket
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(root, "tools", "multi_gpu_check.py")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    assert "with and without peer memory" in r.stdout


def test_config3_population_8192_one_generation():
    """BASELINE config 3 (1M-parameter MLP, population_size = 8192, sigma = 0.02) on however many GPUs this process
    has (one): a fused generation at the default precision; ranks are the permutation the oracle computes from the
    same returns, the update moves theta by ~lr, spot-checked members match the oracle's fp32 forward to 1e-5."""
    dims = [128, 512, 512, 512, 512, 288]
    g = torch.Generator().manual_seed(1234)
    obs, tgt = torch.randn(256, 128, generator=g), torch.randn(256, 288, generator=g)
    torch.manual_seed(0)
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=8192, sigma=0.02, policy_kwargs={"dims": dims},
              agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 26)
    es.log = lambda: None
    assert es._fused and es._precision == "f16" and es._pairs == 4096
    before = es._slots[0].theta.clone()
    es.train(n_steps=1)
    ret = es.population_returns[:, 0]
    assert np.isfinite(ret).all()
    ranks = es._ranks.cpu().numpy()
    np.testing.assert_array_equal(ranks, orc.compute_ranks(ret))
    moved, gr = (es._slots[0].theta - before).abs(), es._grad.abs()
    assert float((moved[gr > 1e-2 * gr.max()] - 0.01).abs().max()) < 1e-5
    pop = es.population_parameters
    for member in (0, 4095, 4096, 8191):
        want = orc.synthetic_return(orc.mlp_forward(pop[member].cpu().numpy(), dims, obs.numpy()), tgt.numpy())
        assert abs(ret[member] - float(want)) < 1e-5 * abs(float(want))
