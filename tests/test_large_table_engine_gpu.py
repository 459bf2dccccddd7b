"""The fused engine on a noise table of 2^31 + 2^22 entries: one ES generation whose pairs include rows past
element 2^31, its returns against the oracle and its gradient against float64 over the rows ``_offsets`` names.

A file of its own, so that the 12 GiB table of test_large_table_gpu.py is freed before the engine allocates its own.
"""
import gc

import numpy as np
import pytest
import torch

from oracle import es_oracle as orc
from conftest import rel_err
from test_api_cpu import MLP as _MLP

pytestmark = pytest.mark.gpu

TABLE_LEN = (1 << 31) + (1 << 22)
GIB = 1 << 30
DIMS, B, P, SIGMA = [4, 64, 64, 2], 256, 64, 0.02
SEED = 745          # generation 0 draws two of its 32 rows past element 2^31 from this table


@pytest.mark.parametrize("precision", ["f16", "fp32"])
def test_fused_generation_on_a_table_past_2_31(precision):
    import estorch_b200 as E
    free, _ = torch.cuda.mem_get_info()
    if free < 6 * TABLE_LEN + 2 * GIB:
        pytest.skip(f"needs {(6 * TABLE_LEN + 2 * GIB) / GIB:.1f} GiB of free device memory for a {TABLE_LEN}-entry "
                    f"noise table and its fp16 copy; {free / GIB:.1f} GiB free")
    torch.cuda.reset_peak_memory_stats()
    rec = {}

    class R(E.ES):
        def log(self):
            rec["returns"] = self.population_returns[:, 0].copy()

    g = torch.Generator().manual_seed(7)
    obs, tgt = torch.randn(B, DIMS[0], generator=g), torch.randn(B, DIMS[-1], generator=g)
    torch.manual_seed(0)
    es = R(_MLP, E.DeviceAgent, torch.optim.Adam, population_size=P, sigma=SIGMA, policy_kwargs={"dims": DIMS},
           agent_kwargs=dict(obs=obs, target=tgt), optimizer_kwargs={"lr": 0.01}, noise_table_size=TABLE_LEN,
           noise_seed=SEED, eval_precision=precision)
    assert es._fused and es._precision == ("f16_any" if precision == "f16" else "fp32")
    assert es._table.numel() == TABLE_LEN
    theta0 = es._slots[0].theta.cpu().numpy().copy()
    es.train(n_steps=1)
    torch.cuda.synchronize()
    n, pairs = theta0.size, P // 2
    offs = es._offsets.clone()
    np.testing.assert_array_equal(offs.cpu().numpy(), orc.noise_offsets(SEED, 0, 0, pairs, TABLE_LEN, n))
    assert int((offs >= 1 << 31).sum()) >= 2, "the precondition: rows past element 2^31"
    # the rows _offsets names, gathered on the device, as a small table at j * n for the oracle
    rows = es._table[offs[:, None] + torch.arange(n, device=offs.device)[None, :]]
    small = rows.cpu().numpy().reshape(-1)
    pop, _ = orc.sample_population(theta0, small, np.arange(pairs) * n, SIGMA)
    got = rec["returns"]
    exact = np.array([orc.synthetic_return(orc.mlp_forward(pop[i], DIMS, obs.numpy()), tgt.numpy())
                      for i in range(P)])
    if precision == "f16":
        emu = np.array([orc.synthetic_return(orc.mlp_forward_f16(pop[i], DIMS, obs.numpy()), tgt.numpy())
                        for i in range(P)])
        assert rel_err(got, emu) < 1e-5
        assert rel_err(got, exact) < 3e-5
    else:
        assert rel_err(got, exact) < 1e-5
    ranks = orc.compute_ranks(got)
    np.testing.assert_array_equal(es._ranks.cpu().numpy(), ranks)
    c = orc.center_values(P).astype(np.float32)[ranks].astype(np.float64)
    want = (c[:pairs] - c[pairs:]) @ rows.double().cpu().numpy() / P
    assert rel_err(es._grad.cpu().numpy(), want) < 1e-5
    print(f"{precision}: peak device memory {torch.cuda.max_memory_allocated() / GIB:.2f} GiB")
    es.close()
    del es, rows
    gc.collect()
    torch.cuda.empty_cache()
