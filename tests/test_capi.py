"""The C-ABI shared library loads and exports every symbol include/estk.h declares
(no compute calls: this runs without a GPU)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "estk.h")).read()
    return sorted(set(re.findall(r"ESTK_API\s+[\w\s\*]+?\b(estk_\w+)\s*\(", text)))


def test_header_and_binding_agree():
    from estorch_b200 import _capi
    declared = _declared_symbols()
    assert len(declared) == 25
    assert sorted(_capi.SIGNATURES) == declared


def test_library_loads_and_exports_the_25_symbols_of_abi_200():
    from estorch_b200 import _capi
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = _capi.load()
    for name in _declared_symbols():
        assert hasattr(lib, name), f"libestk.so does not export {name}"
    assert lib.estk_version() == 200
    assert isinstance(lib.estk_last_error(), bytes)


def test_struct_layouts_match_header():
    import ctypes as C
    from estorch_b200 import _capi
    assert C.sizeof(_capi.EstkState) == 32
    assert C.sizeof(_capi.EstkMlpDesc) == 4 * (1 + 9 + 1)
    assert C.sizeof(_capi.EstkAdamDesc) == 48
    assert _capi.EstkState.best_reward.offset == 20 and _capi.EstkState.improved.offset == 24


def test_product_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from estorch_b200.backend import CudaBackend
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        CudaBackend()


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "estorch_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f


def test_error_reporting_and_precision_probe_without_gpu():
    """estk_ctx_create on a box without a usable device returns a negative status and leaves a
    message in estk_last_error(); null arguments are rejected before any CUDA call."""
    import ctypes as C
    import torch
    from estorch_b200 import _capi
    lib = _capi.load()
    assert lib.estk_ctx_create(0, None) == -1                       # ESTK_ERR_INVALID
    assert b"null" in lib.estk_last_error()
    if not torch.cuda.is_available():
        ctx = C.c_void_p()
        rc = lib.estk_ctx_create(0, C.byref(ctx))
        assert rc < 0 and len(lib.estk_last_error()) > 0 and not ctx.value
    assert lib.estk_ctx_destroy(None) == 0
    assert lib.estk_eval_mlp_supported(None, _capi.ESTK_PREC_BF16, 256) == 0
