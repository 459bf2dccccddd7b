"""ctypes binding of libestk.so (the C ABI declared in include/estk.h).

The library is built in-tree by ``estorch_b200/csrc/build.sh`` (or
``__graft_entry__.build()``).  There is NO fallback: if the shared object is
missing or a call fails, a ``RuntimeError`` is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# ESTK_LIBRARY selects another build of the same library (A/B timing of kernel variants only)
LIB_PATH = os.environ.get("ESTK_LIBRARY") or os.path.join(_HERE, "lib", "libestk.so")

ESTK_MAX_LAYERS = 8
ESTK_MAX_POPULATION = 1 << 22
# estk_mlp_desc.activation bit fields: hidden activation in bits 0-7, output activation in bits 8-15,
# the loss in bits 16-23 (0: squared error)
ESTK_ACT_RELU = 0
ESTK_ACT_TANH = 1
ESTK_ACT_ELU = 3
ESTK_ACT_SILU = 4
ESTK_ACT_LEAKY_RELU = 5
ESTK_ACT_OUT_TANH = 1 << 8
ESTK_LOSS_XENT = 1 << 16
# evaluate precision codes (estk_eval_mlp, estk_eval_conv_vbn)
ESTK_PREC_FP32 = 0
ESTK_PREC_F16 = 1
ESTK_PREC_BF16 = 2
ESTK_PREC_BF16S = 3
ESTK_PREC_F16_ANY = 4


class EstkState(C.Structure):
    """Mirror of ``estk_state`` (32 bytes, device resident)."""
    _fields_ = [("generation", C.c_int64), ("adam_step", C.c_int64),
                ("episode_reward", C.c_float), ("best_reward", C.c_float),
                ("improved", C.c_int32), ("reserved", C.c_int32)]


class EstkMlpDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("dims", C.c_int32 * (ESTK_MAX_LAYERS + 1)),
                ("activation", C.c_int32)]


class EstkAdamDesc(C.Structure):
    _fields_ = [("lr", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double),
                ("eps", C.c_double), ("weight_decay", C.c_double), ("clamp", C.c_float)]


_P = C.c_void_p
_I32, _I64, _U64, _F32 = C.c_int32, C.c_int64, C.c_uint64, C.c_float

# name -> argtypes; every function returns int except estk_last_error (a string) and these:
_INT64_RESULTS = {"estk_eval_conv_vbn_scratch_bytes", "estk_xr_workspace_bytes"}
SIGNATURES = {
    "estk_version": [],
    "estk_last_error": [],
    "estk_ctx_create": [C.c_int, C.POINTER(_P)],
    "estk_ctx_destroy": [_P],
    "estk_ctx_info": [_P, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)],
    "estk_fill_noise_table": [_P, _P, _I64, _U64, _P],
    "estk_make_offsets": [_P, _U64, _P, _I64, _I64, _I32, _I64, _I64, _P, _P, _P],
    "estk_perturb_rows": [_P, _P, _I64, _P, _P, _I32, _F32, _I32, _I32, _P, _P, _P],
    "estk_shadow_f16": [_P, _P, _P, _I64, _P, _P],
    "estk_shadow_bf16": [_P, _P, _P, _I64, _P],
    "estk_eval_mlp": [_P, C.POINTER(EstkMlpDesc), _I32, _P, _P, _P, _P, _P, _P, _I32, _F32, _P, _P, _I32,
                      _P, _P, _P, _P, _I32, _I32, _P, _P],
    "estk_eval_mlp_supported": [C.POINTER(EstkMlpDesc), _I32, _I32],
    "estk_eval_conv_vbn_scratch_bytes": [_P, _I32, _I32, _I32],
    "estk_eval_conv_vbn": [_P, _I32, _I32, _P, _P, _P, _P, _P, _I32, _F32, _P, _I32, _P, _P, _I32, _P, _P, _P, _I64,
                           _P],
    "estk_track_best": [_P, _P, _P, _P, _P, _I64, _P],
    "estk_rank_grad_adam": [_P, _P, _P, _F32, _F32, _I32, _P, _P, _P, _P, _I64, _P, _P, _P, _P,
                            C.POINTER(EstkAdamDesc), _P, _P, _P, _P],
    "estk_rank_grad": [_P, _P, _P, _F32, _F32, _I32, _I32, _P, _P, _P, _P, _I32, _I32, _I64, _P, _P, _P, _P],
    "estk_xr_workspace_bytes": [_I64],
    "estk_peer_alloc": [_P, _I64, C.POINTER(C.c_void_p), C.c_char_p],
    "estk_peer_open": [_P, C.c_char_p, C.POINTER(C.c_void_p)],
    "estk_peer_close": [_P, _P],
    "estk_peer_free": [_P, _P],
    "estk_rank_grad_xr_adam": [_P, _P, _P, _F32, _F32, _I32, _I32, _I32, _P, _P, _P, _I32, _I32, _I64,
                               C.POINTER(C.c_void_p), _P, _P, _P, _P, C.POINTER(EstkAdamDesc), _P, _P, _P, _P],
    "estk_clamp_adam": [_P, _P, _I32, _I64, _P, _P, _P, _P, C.POINTER(EstkAdamDesc), _P, _P],
    "estk_knn_novelty": [_P, _P, _I32, _P, _I32, _I32, _I32, _P, _P],
}

_lib = None


def load():
    """Load libestk.so once; raise loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"estorch_b200: CUDA library not found at {LIB_PATH}. Build it with "
            "`bash estorch_b200/csrc/build.sh` (or `python -c 'import __graft_entry__ as g; "
            "g.build()'`). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.argtypes = argtypes
        fn.restype = (C.c_char_p if name == "estk_last_error" else
                      C.c_int64 if name in _INT64_RESULTS else C.c_int)
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().estk_last_error()
        raise RuntimeError(f"{what} failed (estk_status {rc}): {msg.decode() if msg else '?'}")
