"""C ABI of the evaluate and the launch counter on the H100: the argument checks every precision of
estk_eval_mlp applies before it launches anything, and ``CudaBackend.launches`` against the kernels
the profiler sees in fused generations."""
import glob
import os
import re

import numpy as np
import pytest
import torch

from oracle import es_oracle as orc
from test_activations_cpu import ActMLP
import estorch_b200 as E

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIMS, B = [64, 256, 64], 256


@pytest.fixture(scope="module")
def be():
    from estorch_b200.backend import CudaBackend
    return CudaBackend(torch.device("cuda", 0))


def dev(be, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(be.device)


def _problem(be, pairs=2):
    rng = np.random.RandomState(3)
    n = orc.mlp_param_count(DIMS)
    table = orc.round_f16(rng.standard_normal(n + (1 << 14)).astype(np.float32))
    theta = (rng.standard_normal(n) * 0.05).astype(np.float32)
    obs = rng.standard_normal((B, DIMS[0])).astype(np.float32)
    tgt = rng.standard_normal((B, DIMS[-1])).astype(np.float32)
    offs = orc.noise_offsets(7, 0, 0, pairs, table.size, n)
    return dev(be, theta), dev(be, table), dev(be, offs), dev(be, obs), dev(be, tgt)


def _sixteen_bit(be, mode, theta, table):
    """The 16-bit buffers precision `mode` reads (see include/estk.h, estk_eval_mlp)."""
    if mode == "f16":
        t16 = be.alloc(table.numel(), dtype=torch.float16)
        assert be.shadow_f16(table, t16) == 0
        return {"table16": t16}
    if mode == "bf16s":
        th16, t16 = be.alloc(theta.numel(), dtype=torch.bfloat16), be.alloc(table.numel(), dtype=torch.bfloat16)
        be.shadow_bf16(theta, th16)
        be.shadow_bf16(table, t16)
        return {"theta16": th16, "table16": t16}
    return {}


@pytest.mark.parametrize("mode", ["f16", "bf16", "bf16s"])
def test_tensor_core_bc_outputs_need_positive_bc_obs(be, mode):
    """Behaviour-characteristic outputs with bc_obs = 0 are refused by every precision, before any launch."""
    theta, table, offs, obs, tgt = _problem(be)
    kw = _sixteen_bit(be, mode, theta, table)
    torch.cuda.synchronize()
    ret, bcp, bcm = be.zeros(4).fill_(7.0), be.zeros(2, 256), be.zeros(2, 256)
    launches = be.launches
    with pytest.raises(RuntimeError, match=r"estk_status -1\)"):
        be.eval_mlp(DIMS, theta, table, offs, None, 2, 0.02, obs, tgt, ret[:2], ret[2:], bcp, bcm, 0, 256,
                    precision=mode, **kw)
    torch.cuda.synchronize()
    assert be.launches == launches
    assert torch.equal(ret, torch.full_like(ret, 7.0))


@pytest.mark.parametrize("mode", ["bf16", "bf16s"])
def test_tensor_core_centre_needs_aligned_theta(be, mode):
    """The bf16 / bf16s centre evaluation reads theta with 16-byte loads: an unaligned theta is refused before
    any launch, as it is for f16."""
    theta, table, offs, obs, tgt = _problem(be)
    kw = _sixteen_bit(be, mode, theta, table)
    shifted = be.zeros(theta.numel() + 1)
    shifted[1:].copy_(theta)
    unaligned = shifted[1:]
    assert unaligned.data_ptr() % 16 != 0
    torch.cuda.synchronize()
    one = be.zeros(1).fill_(7.0)
    launches = be.launches
    with pytest.raises(RuntimeError, match=r"estk_status -1\)"):
        be.eval_mlp_center(DIMS, unaligned, obs, tgt, one, precision=mode,
                           **({"theta16": kw["theta16"]} if mode == "bf16s" else {}))
    torch.cuda.synchronize()
    assert be.launches == launches and float(one) == 7.0


def _library_kernels():
    """Names of the kernels libestk defines (every __global__ function of its sources)."""
    names = set()
    for path in glob.glob(os.path.join(ROOT, "estorch_b200", "csrc", "*.cu")):
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)", open(path).read()))
    assert {"eval_mlp_kernel", "eval_mlp_tc_kernel", "rank_grad_kernel", "track_best_kernel"} <= names
    return names


@pytest.mark.parametrize("precision", ["fp32", "f16", "bf16", "bf16s"])
def test_launch_counter_matches_profiled_kernels(monkeypatch, precision):
    """``CudaBackend.launches`` (bench.py's gpu_launches) counts exactly the libestk kernels that eager fused
    generations enqueue: with and without the post-update rollout folded into the evaluate launch."""
    monkeypatch.setenv("ESTORCH_B200_GRAPH", "0")
    g = torch.Generator().manual_seed(5)
    obs, tgt = torch.randn(B, DIMS[0], generator=g), torch.randn(B, DIMS[-1], generator=g)
    torch.manual_seed(5)
    es = E.ES(ActMLP, E.DeviceAgent, torch.optim.Adam, population_size=64, sigma=0.02,
              policy_kwargs={"dims": DIMS, "hidden": "relu"}, agent_kwargs=dict(obs=obs, target=tgt),
              optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 18, log_interval=4, eval_precision=precision)
    assert es._fused and es._precision == precision
    es.log = lambda: None
    es.train(n_steps=1)                 # set-up launches (table copies, shadows) stay outside the window
    torch.cuda.synchronize()
    names = _library_kernels()
    launches0 = es._be.launches
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        es.train(n_steps=3)             # generations 0 and 1 fold their rollout into the next launch (tensor cores)
        torch.cuda.synchronize()
    kernels = [e.name for e in prof.events()
               if e.device_type == torch.autograd.DeviceType.CUDA and any(k in e.name for k in names)]
    print(f"{precision}: {len(kernels)} libestk kernels, counter {es._be.launches - launches0}")
    assert len(kernels) == es._be.launches - launches0 > 0
