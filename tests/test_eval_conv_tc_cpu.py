"""C ABI of the tensor-core conv + VirtualBatchNorm evaluate without a GPU: argument checks
run before any CUDA call, and the ctypes binding matches the header."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_params(name):
    text = open(os.path.join(ROOT, "include", "estk.h")).read()
    m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", text)
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


def test_conv_binding_with_precision_argument_matches_header():
    from estorch_b200 import _capi
    for name in ("estk_eval_conv_vbn", "estk_eval_conv_vbn_scratch_bytes"):
        assert len(_capi.SIGNATURES[name]) == len(_header_params(name)), name
        assert "int32_t precision" in _header_params(name), name
    assert "const uint16_t* table16" in _header_params("estk_eval_conv_vbn")


def test_conv_f16_precision_rejects_null_arguments_before_any_cuda_call():
    from estorch_b200 import _capi
    lib = _capi.load()
    rc = lib.estk_eval_conv_vbn(None, _capi.ESTK_PREC_F16, 4, None, None, None, None, None, 1, 0.02, None, 128, None,
                                None, 32, None, None, None, 0, None)
    assert rc == -1
    assert b"null" in lib.estk_last_error()
    assert lib.estk_eval_conv_vbn_scratch_bytes(None, _capi.ESTK_PREC_F16, 128, 32) == -1
