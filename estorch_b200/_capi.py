"""ctypes binding of libestk.so (the C ABI declared in include/estk.h, include/estk_batch.h,
include/estk_act_cnn.h and include/estk_eval_cnn_tf32.h).

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
# the longest noise table (entries) every kernel reads correctly; estk_make_offsets refuses longer ones
ESTK_MAX_TABLE_LEN = 1 << 34
# estk_mlp_desc.activation bit fields: hidden activation in bits 0-7, output activation in bits 8-15,
# the loss in bits 16-23 (0: squared error; ESTK_ACTIONS: no return, the outputs on each member's own observations)
ESTK_ACT_RELU = 0
ESTK_ACT_TANH = 1
ESTK_ACT_ELU = 3
ESTK_ACT_SILU = 4
ESTK_ACT_LEAKY_RELU = 5
# recurrent cells in the hidden field, with ESTK_ACTIONS only: one GRUCell / LSTMCell step + a Linear head
ESTK_CELL_GRU = 8
ESTK_CELL_LSTM = 9
ESTK_ACT_OUT_TANH = 1 << 8
ESTK_LOSS_XENT = 1 << 16
ESTK_ACTIONS = 3 << 16
# the return is the fraction of rows whose logits' first argmax is the target's first argmax (fp32)
ESTK_LOSS_ACCURACY = 6 << 16
# bits 24-31: n_conv, the number of leading Conv2d layers of a convolutional policy (the CNN evaluate, fp32);
# its dims[0] is ESTK_CNN_INPUT(c, h, w) and dims[1..n_conv] ESTK_CNN_CONV(out_c, k, stride, pad)
ESTK_CNN_SHIFT = 24
ESTK_CNN_MAX_CONV = 7


def ESTK_CNN_N_CONV(n):
    return int(n) << ESTK_CNN_SHIFT


def ESTK_CNN_INPUT(c, h, w):
    return int(c) | int(h) << 10 | int(w) << 20


def ESTK_CNN_CONV(out_c, k, stride, pad):
    return int(out_c) | int(k) << 12 | int(stride) << 18 | int(pad) << 24

# estk_eval_conv_vbn with n_actions | ESTK_ACTIONS: VBN statistics per member, in floats
ESTK_CONV_VBN_STATS_FLOATS = 17984
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

# include/estk_batch.h: the minibatch sampler, declared beside the core of estk.h
BATCH_SIGNATURES = {
    "estk_sample_batch": [_P, _U64, _P, _I64, _I64, _I32, _P, _I64, _P, _P, _I64, _P, _P, _P],
}

# include/estk_act_cnn.h: population mode for convolutional policies, declared beside the core of estk.h
ACT_CNN_SIGNATURES = {
    "estk_act_cnn": [_P, C.POINTER(EstkMlpDesc), _P, _P, _P, _P, _I32, _F32, _P, _I32, _P, _P, _P],
}

# include/estk_eval_cnn_tf32.h: the convolutional evaluate on TF32 tensor cores, declared beside the core of estk.h
EVAL_CNN_TF32_SIGNATURES = {
    "estk_eval_cnn_tf32": [_P, C.POINTER(EstkMlpDesc), _P, _P, _P, _P, _I32, _F32, _P, _P, _I32, _P, _P, _P, _P,
                           _I32, _I32, _P],
    "estk_eval_cnn_tf32_supported": [C.POINTER(EstkMlpDesc), _I32],
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
    for name, argtypes in {**SIGNATURES, **BATCH_SIGNATURES, **ACT_CNN_SIGNATURES,
                           **EVAL_CNN_TF32_SIGNATURES}.items():
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
