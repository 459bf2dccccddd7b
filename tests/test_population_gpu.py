"""Population mode on the H100: estk_eval_mlp with ESTK_ACTIONS (estk_eval_mlp_act.cu) bit-identical to
the fp32 evaluate's behaviour characteristic, its determinism, member isolation, agreement with a torch
forward of materialised rows, refusals before launch, ES / NSR-ES in population mode against the reference
goldens, and a CartPole population that learns."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA GPU", allow_module_level=True)

from estorch_b200 import _capi  # noqa: E402
from estorch_b200.backend import CudaBackend, mlp_desc  # noqa: E402
import test_population_cpu as cpu  # noqa: E402

ACTIONS = _capi.ESTK_ACTIONS
CODES = [h | o for h in (0, 1, 3, 4, 5) for o in (0, 1 << 8)]


@pytest.fixture(scope="module")
def be():
    return CudaBackend()


def _setup(be, dims, pairs, seed=0, scale=0.3):
    g = torch.Generator(device="cpu").manual_seed(seed)
    n = sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))
    theta = ((torch.rand(n, generator=g) * 2 - 1) * scale / np.sqrt(max(dims[:-1]))).to(be.device)
    table = be.alloc(max(1 << 16, (n + 31) // 32 * 32 + 32 * 4096))
    be.fill_noise_table(table, 11 + seed)
    t16 = be.alloc(table.numel(), dtype=torch.float16)
    assert be.shadow_f16(table, t16) == 0
    offsets, order = be.zeros(pairs, dtype=torch.int64), be.zeros(pairs, dtype=torch.int32)
    be.make_offsets(5 + seed, None, 0, 0, pairs, table.numel(), n, offsets, order)
    return theta, table, t16, offsets, order


def _bc_reference(be, dims, code, theta, table, offsets, pairs, sigma, obs):
    """estk_eval_mlp FP32 with the squared error: its behaviour characteristic, every member on ``obs``."""
    B, out = obs.shape[0], dims[-1]
    bp, bm = be.zeros(pairs, B * out), be.zeros(pairs, B * out)
    rp, rm = be.zeros(pairs), be.zeros(pairs)
    be.eval_mlp(dims, theta, table, offsets, None, pairs, sigma, obs, be.zeros(B, out), rp, rm, bp, bm, B, B * out,
                precision="fp32", act=code)
    return torch.cat([bp, bm]).view(2 * pairs, B, out)


def _act(be, dims, code, theta, table, offsets, pairs, sigma, obs3, order=None, table16=None):
    out = be.alloc(obs3.shape[0], obs3.shape[1], dims[-1])
    be.act_mlp(dims, theta, None if table16 is not None else table, offsets, order, pairs, sigma, obs3, out,
               act=code, table16=table16)
    return out


@pytest.mark.parametrize("code", CODES)
def test_act_is_bit_identical_to_the_fp32_behaviour_characteristic_for_every_code(be, code):
    dims, pairs, B, sigma = [17, 33, 5], 7, 3, 0.05
    theta, table, t16, offsets, order = _setup(be, dims, pairs)
    obs = torch.randn(B, dims[0], device=be.device) * 2
    ref = _bc_reference(be, dims, code, theta, table, offsets, pairs, sigma, obs)
    got = _act(be, dims, code, theta, table, offsets, pairs, sigma, obs.expand(2 * pairs, B, dims[0]).contiguous())
    assert torch.equal(got, ref)


SHAPES = [([4, 64, 64, 2], (1, 3, 16, 100), (1, 7, 2048)),
          ([17, 33, 5], (1, 3, 16, 100), (1, 7, 2048)),
          ([24, 64, 64, 4], (1, 3), (2048,)),
          ([1100, 1100, 8], (1, 3, 16, 100), (1, 7))]       # B >= 16 here streams through the context slab


@pytest.mark.parametrize("dims,Bs,pairs_list", SHAPES, ids=lambda v: "-".join(map(str, v)) if isinstance(v, list) else None)
def test_act_is_bit_identical_across_shapes_batches_and_populations(be, dims, Bs, pairs_list):
    for i, (B, pairs) in enumerate([(B, p) for B in Bs for p in pairs_list]):
        code = CODES[i % len(CODES)]
        theta, table, t16, offsets, order = _setup(be, dims, pairs, seed=i)
        obs = torch.randn(B, dims[0], device=be.device)
        ref = _bc_reference(be, dims, code, theta, table, offsets, pairs, 0.02, obs)
        got = _act(be, dims, code, theta, table, offsets, pairs, 0.02, obs.expand(2 * pairs, B, dims[0]).contiguous(),
                   order=order, table16=t16 if i % 2 else None)
        assert torch.equal(got, ref), (dims, B, pairs, hex(code))
        # the centre: theta's outputs, bit-identical to the centre evaluate's behaviour characteristic
        bc = be.zeros(B * dims[-1])
        be.eval_mlp_center(dims, theta, obs, be.zeros(B, dims[-1]), be.zeros(1), bc, B, B * dims[-1], act=code)
        out = be.alloc(1, B, dims[-1])
        be.act_mlp(dims, theta, None, None, None, 1, 0.0, obs[None].contiguous(), out, act=code)
        assert torch.equal(out.view(-1), bc)


def test_same_bits_run_to_run_with_and_without_order_from_either_table(be):
    dims, pairs, B = [24, 64, 64, 4], 300, 2
    theta, table, t16, offsets, order = _setup(be, dims, pairs)
    obs = torch.randn(2 * pairs, B, dims[0], device=be.device)
    outs = [_act(be, dims, 0x104, theta, table, offsets, pairs, 0.05, obs, order=o, table16=t)
            for o in (None, order) for t in (None, t16) for _ in range(2)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_members_are_isolated(be):
    dims, pairs, B = [17, 33, 5], 64, 3
    theta, table, _, offsets, order = _setup(be, dims, pairs)
    obs = torch.randn(2 * pairs, B, dims[0], device=be.device)
    a = _act(be, dims, 3, theta, table, offsets, pairs, 0.05, obs, order=order)
    keep = torch.tensor([0, 5, pairs, pairs + 63], device=be.device)
    obs2 = torch.randn_like(obs) * 10
    obs2[keep] = obs[keep]
    b = _act(be, dims, 3, theta, table, offsets, pairs, 0.05, obs2, order=order)
    assert torch.equal(a[keep], b[keep])
    assert not torch.equal(a, b)


@pytest.mark.parametrize("code", [0, 1 | (1 << 8), 4])
def test_act_agrees_with_a_torch_forward_of_materialised_rows(be, code):
    dims, pairs, B, sigma = [24, 64, 64, 4], 128, 3, 0.05
    theta, table, _, offsets, _ = _setup(be, dims, pairs)
    obs = torch.randn(2 * pairs, B, dims[0], device=be.device)
    got = _act(be, dims, code, theta, table, offsets, pairs, sigma, obs).double()
    rows = be.alloc(2 * pairs, theta.numel())
    be.perturb_rows(theta, table, offsets, pairs, sigma, 0, 2 * pairs, rows)
    h, idx = obs.double(), 0
    hidden = {0: torch.relu, 1: torch.tanh, 4: torch.nn.functional.silu}[code & 0xff]
    for li in range(len(dims) - 1):
        i, o = dims[li], dims[li + 1]
        W = rows[:, idx: idx + i * o].double().view(-1, o, i)
        b = rows[:, idx + i * o: idx + i * o + o].double()
        idx += i * o + o
        h = torch.bmm(h, W.transpose(1, 2)) + b[:, None, :]
        if li + 2 < len(dims):
            h = hidden(h)
    if code & (1 << 8):
        h = torch.tanh(h)
    assert float((got - h).abs().max() / h.abs().max()) < 1e-6


def test_refusals_happen_before_any_launch(be):
    lib = be.lib
    dims, pairs, B = [17, 33, 5], 7, 3
    theta, table, t16, offsets, order = _setup(be, dims, pairs)
    obs = torch.randn(2 * pairs, B, dims[0], device=be.device)
    out = be.zeros(2 * pairs, B, dims[-1])
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    minus = C.c_void_p(out.data_ptr() + pairs * B * dims[-1] * 4)

    def call(code, precision, bc_plus):
        d = mlp_desc(dims, code)
        return lib.estk_eval_mlp(be._ctx, C.byref(d), precision, p(theta), p(theta), p(table), p(t16), p(offsets),
                                 p(order), pairs, 0.05, p(obs), None, B, None, None, bc_plus, minus, B,
                                 B * dims[-1], None, be._stream())
    for prec in (_capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S, _capi.ESTK_PREC_F16_ANY):
        assert call(ACTIONS, prec, p(out)) == -3                                   # ESTK_ERR_UNSUPPORTED
    for code in (0x30002, 0x30200, 0x20000 | 0x100, 0x70000):
        assert call(code, _capi.ESTK_PREC_FP32, p(out)) == -1                     # ESTK_ERR_INVALID
    assert call(ACTIONS, _capi.ESTK_PREC_FP32, None) == -1
    torch.cuda.synchronize()
    assert float(out.abs().sum()) == 0.0                                          # nothing was written
    assert call(ACTIONS, _capi.ESTK_PREC_FP32, p(out)) == 0


def test_es_population_mode_matches_reference_golden(be):
    cpu.check_es_golden(*cpu.run_es_golden(be))


def test_nsr_population_mode_matches_reference_golden(be):
    cpu.check_nsr_golden(*cpu.run_nsr_golden(be))


def test_cartpole_population_learns(be):
    spec = importlib.util.spec_from_file_location("vector_cartpole", os.path.join(ROOT, "examples", "vector_cartpole.py"))
    vc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(vc)
    from estorch_b200 import ES
    torch.manual_seed(0)
    means = []
    es = ES(vc.Policy, vc.VectorCartPole, torch.optim.Adam, population_size=1024, sigma=0.02,
            optimizer_kwargs={"lr": 0.03}, noise_table_size=1 << 22, noise_seed=3, _backend=be)
    es.log = lambda: means.append(float(es.population_returns.mean()))
    assert es._population
    es.train(n_steps=20)
    assert len(means) == 20
    assert np.mean(means[-3:]) > np.mean(means[:3]) + 20, means
