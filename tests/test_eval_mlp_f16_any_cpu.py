"""ESTK_PREC_F16_ANY without a GPU: the header and the binding agree on the code, the support probe and the
argument checks of the C ABI, and the precision ES picks for eval_precision="f16" / "auto" / "bf16" on
shapes inside and outside the cluster kernel's rule (with a stand-in backend built on the oracle)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import _mlp_oracle as mlp
from _mlp_oracle import MLP
from _oracle_backend import OracleBackend
import estorch_b200 as E
from estorch_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


def _supported(lib, dims, code, precision, B):
    from estorch_b200.backend import mlp_desc
    d = mlp_desc(dims, code)
    return lib.estk_eval_mlp_supported(C.byref(d), precision, B)


def test_header_and_binding_agree_on_the_code():
    header = open(os.path.join(ROOT, "include", "estk.h")).read()
    m = re.search(r"#define\s+ESTK_PREC_F16_ANY\s+(\d+)", header)
    assert m and int(m.group(1)) == _capi.ESTK_PREC_F16_ANY == 4
    assert re.search(r"#define\s+ESTK_VERSION\s+200\b", header)
    from estorch_b200.backend import _PRECISIONS
    assert _PRECISIONS["f16_any"] == (4, torch.float16)


def test_support_probe_serves_every_shape_and_leaves_f16_unchanged():
    lib = _lib()
    F16_ANY = _capi.ESTK_PREC_F16_ANY
    assert _supported(lib, [784, 100, 10], mlp.LOSS_XENT, F16_ANY, 100) == 1
    assert _supported(lib, [3072, 512, 10], mlp.LOSS_XENT, F16_ANY, 256) == 1
    assert _supported(lib, [4, 64, 64, 2], 0, F16_ANY, 1) == 1
    assert _supported(lib, [1, 1], mlp.ACT_TANH | mlp.ACT_OUT_TANH, F16_ANY, 60000) == 1
    assert _supported(lib, [128, 512, 512, 288], 0, F16_ANY, 256) == 1           # a rule shape too
    for code in (2, 0x200, 0x10101, 0x20000, 0x10200, 0x10100, 0x1000000, 0x10002):
        assert _supported(lib, [784, 100, 10], code, F16_ANY, 100) == 0, hex(code)
    assert _supported(lib, [784, 100, 10], 0, F16_ANY, 0) == 0
    assert _supported(lib, [784, 0, 10], 0, F16_ANY, 100) == 0
    assert lib.estk_eval_mlp_supported(None, F16_ANY, 100) == 0
    for prec in (_capi.ESTK_PREC_F16, _capi.ESTK_PREC_BF16, _capi.ESTK_PREC_BF16S):
        assert _supported(lib, [784, 100, 10], 0, prec, 100) == 0
        assert _supported(lib, [64, 64, 32], 0, prec, 100) == 0
        assert _supported(lib, [64, 64, 32], 0, prec, 256) == 1
    assert _supported(lib, [320, 64, 32], 0, _capi.ESTK_PREC_F16, 256) == 0
    assert _supported(lib, [64, 64, 10], mlp.LOSS_XENT, _capi.ESTK_PREC_F16, 256) == 0
    for prec in (_capi.ESTK_PREC_FP32, 5, -1):
        assert _supported(lib, [64, 64, 32], 0, prec, 256) == 0


def test_null_arguments_are_refused_before_any_cuda_call():
    from estorch_b200.backend import mlp_desc
    lib = _lib()
    d = mlp_desc([784, 100, 10], mlp.LOSS_XENT)
    fake = C.c_void_p(16)                    # never dereferenced: the checks fail first
    args = dict(ctx=fake, desc=C.byref(d), theta=fake, theta16=None, table=fake, table16=fake, offsets=fake,
                obs=fake, target=fake, rp=fake, rm=fake)

    def call(**over):
        a = {**args, **over}
        return lib.estk_eval_mlp(a["ctx"], a["desc"], _capi.ESTK_PREC_F16_ANY, a["theta"], a["theta16"], a["table"],
                                 a["table16"], a["offsets"], None, 2, 0.02, a["obs"], a["target"], 100, a["rp"],
                                 a["rm"], None, None, 0, 0, None, None)
    for name in ("ctx", "desc", "theta", "table", "table16", "obs", "target", "rp", "rm"):
        assert call(**{name: None}) == -1, name
    assert "null argument" in lib.estk_last_error().decode()


# ------------------------------------------------------------------ ES routing with a stand-in backend
class AnyShapeBackend(OracleBackend):
    """Stand-in that records the evaluate precisions; ``with_f16_any=False`` answers no to every "f16_any" probe."""

    def __init__(self, with_f16_any=True):
        super().__init__(tensor_core=True)
        self.precisions = set()
        if not with_f16_any:
            self.eval_supports_f16_any = lambda dims, B, act=0: False

    def eval_mlp(self, *a, precision="fp32", centre_out=None, **kw):
        self.precisions.add(precision)
        if precision == "f16_any":
            assert centre_out is None
        return super().eval_mlp(*a, precision=precision, centre_out=centre_out, **kw)

    def eval_mlp_center(self, *a, precision="fp32", **kw):
        self.precisions.add(precision)
        return super().eval_mlp_center(*a, precision=precision, **kw)


def _es(dims, B, eval_precision, loss="cross_entropy", be=None):
    rng = np.random.RandomState(3)
    obs = torch.from_numpy(rng.standard_normal((B, dims[0])).astype(np.float32))
    tgt = torch.from_numpy(np.eye(dims[-1], dtype=np.float32)[rng.randint(0, dims[-1], B)])
    be = be or AnyShapeBackend()
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.05, policy_kwargs={"dims": dims},
              agent_kwargs=dict(obs=obs, target=tgt, loss=loss), optimizer_kwargs={"lr": 0.01},
              noise_table_size=1 << 16, eval_precision=eval_precision, _backend=be)
    es.log = lambda: None
    return es, be, obs, tgt


OFF_RULE, ON_RULE = ([24, 20, 10], 100), ([64, 64, 32], 256)


def test_f16_off_rule_selects_f16_any_without_deferred_centre_and_trains():
    es, be, obs, tgt = _es(*OFF_RULE, "f16")
    assert es._fused and es._precision == "f16_any"
    es._log_interval = 10                   # a deferred centre would need log() to be skipped
    es.train(n_steps=3)
    assert be.precisions == {"f16_any"} and be.centre_folds == 0
    assert not es._defers_centre()
    with torch.no_grad():
        want = float(torch.nn.functional.cross_entropy(es.policy(obs), tgt))
    assert abs(es.episode_reward + want) < 1e-4 * abs(want)


def test_f16_on_rule_and_auto_are_unchanged():
    assert _es(*ON_RULE, "f16")[0]._precision == "f16"
    assert _es(*ON_RULE, "auto")[0]._precision == "f16"
    assert _es(*OFF_RULE, "auto")[0]._precision == "fp32"
    assert _es(*OFF_RULE, "fp32")[0]._precision == "fp32"
    assert _es(*OFF_RULE, "f16", loss="mse")[0]._precision == "f16_any"


@pytest.mark.parametrize("mode", ["bf16", "bf16s"])
def test_bf16_off_rule_still_raises(mode):
    with pytest.raises(ValueError, match="multiples of 64"):
        _es(*OFF_RULE, mode)


def test_backend_refusing_f16_any_behaves_as_before():
    """A backend whose f16_any probe answers no: off-rule "f16" is refused, on-rule "f16" keeps the cluster kernel."""
    with pytest.raises(ValueError, match="multiples of 64"):
        _es(*OFF_RULE, "f16", be=AnyShapeBackend(with_f16_any=False))
    assert _es(*ON_RULE, "f16", be=AnyShapeBackend(with_f16_any=False))[0]._precision == "f16"


def test_f16_any_reads_the_exact_fp16_table():
    es, be, _, _ = _es(*OFF_RULE, "f16")
    kw = es._eval_kw(es._slots[0])
    assert kw["precision"] == "f16_any" and kw["table16"].dtype == torch.float16
    assert torch.equal(kw["table16"].float(), es._table)
    assert "table16" not in es._eval_kw(es._slots[0], centre=True)
