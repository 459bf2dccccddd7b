"""Status codes of refused estk_eval_mlp and estk_eval_conv_vbn calls, without a GPU.

Each row is one call and the estk_status it returns.  Which back end an activation code reaches, and the
order in which that back end checks precision, pointers, sizes and packed fields, decide between
ESTK_ERR_INVALID (I) and ESTK_ERR_UNSUPPORTED (U).  Every call here is refused before the library reads
the context, so a fake non-null pointer stands in for it and for every buffer (none is dereferenced)."""
import ctypes as C
import os

import pytest

from estorch_b200 import _capi

I, U = -1, -3
FAKE = C.c_void_p(256)            # 16-byte aligned, never dereferenced
ODD = C.c_void_p(260)             # not 16-byte aligned
MAX_PAIRS = _capi.ESTK_MAX_POPULATION // 2
GRU, LSTM, ACTIONS, XENT = _capi.ESTK_CELL_GRU, _capi.ESTK_CELL_LSTM, _capi.ESTK_ACTIONS, _capi.ESTK_LOSS_XENT
OUT_TANH, N_CONV = _capi.ESTK_ACT_OUT_TANH, _capi.ESTK_CNN_N_CONV
CNN_IN, CNN_CONV = _capi.ESTK_CNN_INPUT(1, 8, 8), _capi.ESTK_CNN_CONV(2, 3, 1, 0)

ROUTES = {   # route -> (n_layers, dims, activation code) of a well-formed call; the sequence's dims[3] is T
    "dense": (2, (4, 8, 2), 0),
    "actions": (2, (4, 8, 2), ACTIONS),
    "cell": (2, (4, 8, 2), GRU | ACTIONS),
    "sequence": (2, (4, 8, 2, 3), GRU),
    "cnn": (2, (CNN_IN, CNN_CONV, 4), N_CONV(1)),
}


def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


def _eval_mlp(route, centre, **over):
    """estk_eval_mlp on a well-formed call of ``route`` (a population, or the centre: offsets NULL) with the
    arguments in ``over`` replaced."""
    n_layers, dims, code = ROUTES[route]
    a = dict(ctx=FAKE, desc=True, n_layers=n_layers, dims=dims, code=code, precision=0, theta=FAKE, theta16=FAKE,
             table=FAKE, table16=FAKE, offsets=None if centre else FAKE, order=FAKE, pairs=2, sigma=0.02, obs=FAKE,
             target=FAKE, B=4, returns_plus=FAKE, returns_minus=FAKE, bc_plus=None, bc_minus=None, bc_obs=0,
             bc_dim=0, centre_return_out=None)
    if route in ("actions", "cell"):   # the outputs are the bc buffers; there is no return
        a.update(target=None, returns_plus=None, returns_minus=None, bc_plus=FAKE, bc_minus=FAKE, bc_obs=4, bc_dim=8)
    a.update(over)
    d = _capi.EstkMlpDesc()
    d.n_layers = a["n_layers"]
    for i, w in enumerate(a["dims"]):
        d.dims[i] = C.c_int32(w).value
    d.activation = C.c_int32(a["code"]).value
    return _lib().estk_eval_mlp(
        a["ctx"], C.byref(d) if a["desc"] else None, a["precision"], a["theta"], a["theta16"],
        a["table"], a["table16"], a["offsets"], a["order"], a["pairs"], a["sigma"], a["obs"], a["target"], a["B"],
        a["returns_plus"], a["returns_minus"], a["bc_plus"], a["bc_minus"], a["bc_obs"], a["bc_dim"],
        a["centre_return_out"], None)


def _eval_conv_vbn(actions, centre, **over):
    """estk_eval_conv_vbn on a well-formed call (the VBN evaluate, or ESTK_ACTIONS with both phases)."""
    a = dict(ctx=FAKE, precision=0, n_actions=6 | ACTIONS if actions else 6, theta=FAKE, table=FAKE, table16=FAKE,
             offsets=None if centre else FAKE, order=FAKE, pairs=2, sigma=0.02, xref=FAKE, ref_batch=8, obs=FAKE,
             target=None if actions else FAKE, B=4, returns_plus=FAKE, returns_minus=FAKE, scratch=FAKE,
             scratch_bytes=1 << 40)
    a.update(over)
    return _lib().estk_eval_conv_vbn(
        a["ctx"], a["precision"], a["n_actions"], a["theta"], a["table"], a["table16"], a["offsets"], a["order"],
        a["pairs"], a["sigma"], a["xref"], a["ref_batch"], a["obs"], a["target"], a["B"], a["returns_plus"],
        a["returns_minus"], a["scratch"], a["scratch_bytes"], None)


# Each table line: the arguments a call changes from the well-formed one, then for each column the status
# of the centre call (offsets NULL) and of the population call.  "." marks a call that is not refused
# (it would reach the context), so it is not made here.
NAMES = dict(NULL=None, FAKE=FAKE, ODD=ODD, MAX_PAIRS=MAX_PAIRS, GRU=GRU, LSTM=LSTM, ACTIONS=ACTIONS, XENT=XENT,
             OUT_TANH=OUT_TANH, N_CONV=N_CONV, IN=_capi.ESTK_CNN_INPUT, CONV=_capi.ESTK_CNN_CONV, CNN_IN=CNN_IN,
             CNN_CONV=CNN_CONV)

MLP_COLUMNS = tuple(ROUTES)
MLP_ROWS = """
precision=0 B=0                                          | II II II II II
precision=1 B=0                                          | UU UU UU UU UU
precision=2 B=0                                          | UU UU UU UU UU
precision=3 B=0                                          | UU UU UU UU UU
precision=4 B=0                                          | UU UU UU UU UU
precision=7 B=0                                          | II II II II II
precision=-1                                             | II II II II II
precision=7                                              | II II II II II
precision=5 pairs=0                                      | II II II II II
precision=0 centre_return_out=FAKE                       | IU II II UU UU
precision=1 centre_return_out=FAKE                       | IU UU UU UU UU
precision=2 centre_return_out=FAKE                       | IU UU UU UU UU
precision=3 centre_return_out=FAKE                       | IU UU UU UU UU
precision=4 centre_return_out=FAKE                       | IU UU UU UU UU
precision=7 centre_return_out=FAKE                       | II II II II II
precision=0 centre_return_out=FAKE B=0                   | IU II II UU UU
precision=1 centre_return_out=FAKE B=0                   | IU UU UU UU UU
precision=4 centre_return_out=FAKE B=0                   | IU UU UU UU UU
B=0                                                      | II II II II II
B=-1                                                     | II II II II II
pairs=0                                                  | .I .I .I .I .I
pairs=-1                                                 | .I .I .I .I .I
pairs=MAX_PAIRS+1                                        | .I .I .I .I .I
precision=1 B=-1                                         | UU UU UU UU UU
precision=1 pairs=0                                      | UU UU UU UU UU
precision=1 pairs=-1                                     | UU UU UU UU UU
precision=1 pairs=MAX_PAIRS+1                            | UU UU UU UU UU
precision=1 pairs=MAX_PAIRS                              | UU UU UU UU UU
precision=4 B=-1                                         | UU UU UU UU UU
precision=4 pairs=0                                      | .I UU UU UU UU
precision=4 pairs=-1                                     | .I UU UU UU UU
precision=4 pairs=MAX_PAIRS+1                            | .I UU UU UU UU
precision=4 pairs=MAX_PAIRS                              | .. UU UU UU UU
ctx=NULL                                                 | II II II II II
desc=NULL                                                | II II II II II
theta=NULL                                               | II II II II II
table=NULL                                               | .I .. .. .I .I
obs=NULL                                                 | II II II II II
target=NULL                                              | II .. .. II II
returns_plus=NULL                                        | II .. .. II II
returns_minus=NULL                                       | .I .. .. .I .I
bc_plus=NULL                                             | .. II II .. ..
bc_minus=NULL                                            | .. .I .I .. ..
ctx=NULL B=0                                             | II II II II II
desc=NULL B=0                                            | II II II II II
theta=NULL B=0                                           | II II II II II
theta16=NULL B=0                                         | II II II II II
table=NULL B=0                                           | II II II II II
table16=NULL B=0                                         | II II II II II
order=NULL B=0                                           | II II II II II
obs=NULL B=0                                             | II II II II II
target=NULL B=0                                          | II II II II II
returns_plus=NULL B=0                                    | II II II II II
returns_minus=NULL B=0                                   | II II II II II
bc_plus=NULL B=0                                         | II II II II II
bc_minus=NULL B=0                                        | II II II II II
ctx=NULL precision=1                                     | II UU UU UU UU
desc=NULL precision=1                                    | II II II II II
theta=NULL precision=1                                   | II UU UU UU UU
theta16=NULL precision=1                                 | UU UU UU UU UU
table=NULL precision=1                                   | UI UU UU UU UU
table16=NULL precision=1                                 | UI UU UU UU UU
order=NULL precision=1                                   | UU UU UU UU UU
obs=NULL precision=1                                     | II UU UU UU UU
target=NULL precision=1                                  | II UU UU UU UU
returns_plus=NULL precision=1                            | II UU UU UU UU
returns_minus=NULL precision=1                           | UI UU UU UU UU
bc_plus=NULL precision=1                                 | UU UU UU UU UU
bc_minus=NULL precision=1                                | UU UU UU UU UU
ctx=NULL precision=3                                     | II UU UU UU UU
desc=NULL precision=3                                    | II II II II II
theta=NULL precision=3                                   | II UU UU UU UU
theta16=NULL precision=3                                 | II UU UU UU UU
table=NULL precision=3                                   | UI UU UU UU UU
table16=NULL precision=3                                 | UI UU UU UU UU
order=NULL precision=3                                   | UU UU UU UU UU
obs=NULL precision=3                                     | II UU UU UU UU
target=NULL precision=3                                  | II UU UU UU UU
returns_plus=NULL precision=3                            | II UU UU UU UU
returns_minus=NULL precision=3                           | UI UU UU UU UU
bc_plus=NULL precision=3                                 | UU UU UU UU UU
bc_minus=NULL precision=3                                | UU UU UU UU UU
ctx=NULL precision=4                                     | II UU UU UU UU
desc=NULL precision=4                                    | II II II II II
theta=NULL precision=4                                   | II UU UU UU UU
theta16=NULL precision=4                                 | .. UU UU UU UU
table=NULL precision=4                                   | .I UU UU UU UU
table16=NULL precision=4                                 | .I UU UU UU UU
order=NULL precision=4                                   | .. UU UU UU UU
obs=NULL precision=4                                     | II UU UU UU UU
target=NULL precision=4                                  | II UU UU UU UU
returns_plus=NULL precision=4                            | II UU UU UU UU
returns_minus=NULL precision=4                           | .I UU UU UU UU
bc_plus=NULL precision=4                                 | .. UU UU UU UU
bc_minus=NULL precision=4                                | .. UU UU UU UU
bc_plus=FAKE bc_minus=NULL bc_obs=4 bc_dim=8             | .I .I .I .I .I
bc_plus=NULL bc_minus=FAKE                               | .I II II .I .I
bc_plus=FAKE bc_minus=FAKE bc_obs=0 bc_dim=8             | II II II II II
bc_plus=FAKE bc_minus=FAKE bc_obs=4 bc_dim=0             | II II II II II
bc_plus=FAKE bc_minus=NULL bc_obs=4 bc_dim=8 B=0         | II II II II II
bc_plus=NULL bc_minus=FAKE B=0                           | II II II II II
bc_plus=FAKE bc_minus=FAKE bc_obs=0 bc_dim=8 B=0         | II II II II II
bc_plus=FAKE bc_minus=FAKE bc_obs=4 bc_dim=0 B=0         | II II II II II
bc_plus=FAKE bc_minus=NULL bc_obs=4 bc_dim=8 precision=1 | UI UU UU UU UU
bc_plus=NULL bc_minus=FAKE precision=1                   | UI UU UU UU UU
bc_plus=FAKE bc_minus=FAKE bc_obs=0 bc_dim=8 precision=1 | II UU UU UU UU
bc_plus=FAKE bc_minus=FAKE bc_obs=4 bc_dim=0 precision=1 | II UU UU UU UU
bc_plus=FAKE bc_minus=NULL bc_obs=4 bc_dim=8 precision=3 | UI UU UU UU UU
bc_plus=NULL bc_minus=FAKE precision=3                   | UI UU UU UU UU
bc_plus=FAKE bc_minus=FAKE bc_obs=0 bc_dim=8 precision=3 | II UU UU UU UU
bc_plus=FAKE bc_minus=FAKE bc_obs=4 bc_dim=0 precision=3 | II UU UU UU UU
theta=ODD precision=1                                    | II UU UU UU UU
theta16=ODD precision=1                                  | UU UU UU UU UU
table=ODD precision=1                                    | UI UU UU UU UU
table16=ODD precision=1                                  | UI UU UU UU UU
obs=ODD precision=1                                      | II UU UU UU UU
target=ODD precision=1                                   | II UU UU UU UU
theta=ODD precision=3                                    | II UU UU UU UU
theta16=ODD precision=3                                  | II UU UU UU UU
table=ODD precision=3                                    | UI UU UU UU UU
table16=ODD precision=3                                  | UI UU UU UU UU
obs=ODD precision=3                                      | II UU UU UU UU
target=ODD precision=3                                   | II UU UU UU UU
theta=ODD precision=4                                    | II UU UU UU UU
theta16=ODD precision=4                                  | .. UU UU UU UU
table=ODD precision=4                                    | .I UU UU UU UU
table16=ODD precision=4                                  | .I UU UU UU UU
obs=ODD precision=4                                      | II UU UU UU UU
target=ODD precision=4                                   | II UU UU UU UU
code=2                                                   | II II II II II
code=2 B=0                                               | II II II II II
code=2 precision=1                                       | UU II II UU UU
code=2 precision=4                                       | UU II II UU UU
code=6                                                   | II II II II II
code=6 B=0                                               | II II II II II
code=6 precision=1                                       | UU II II UU UU
code=6 precision=4                                       | UU II II UU UU
code=0x200                                               | II II II II II
code=0x200 B=0                                           | II II II II II
code=0x200 precision=1                                   | UU II II UU UU
code=0x200 precision=4                                   | UU II II UU UU
code=0x20000                                             | II II II II II
code=0x20000 B=0                                         | II II II II II
code=0x20000 precision=1                                 | UU II II UU UU
code=0x20000 precision=4                                 | UU II II UU UU
code=0x10100                                             | II II II II II
code=0x10100 B=0                                         | II II II II II
code=0x10100 precision=1                                 | UU II II UU UU
code=0x10100 precision=4                                 | UU II II UU UU
code=0x10101                                             | II II II II II
code=0x10101 B=0                                         | II II II II II
code=0x10101 precision=1                                 | UU II II UU UU
code=0x10101 precision=4                                 | UU II II UU UU
code=2|ACTIONS                                           | II II II II II
code=2|ACTIONS B=0                                       | II II II II II
code=2|ACTIONS precision=1                               | UU II II UU UU
code=2|ACTIONS precision=4                               | UU II II UU UU
code=GRU|XENT|OUT_TANH                                   | II II II II II
code=GRU|XENT|OUT_TANH B=0                               | II II II II II
code=GRU|XENT|OUT_TANH precision=1                       | UU II II UU UU
code=GRU|XENT|OUT_TANH precision=4                       | UU II II UU UU
code=GRU|0x200                                           | II II II II II
code=GRU|0x200 B=0                                       | II II II II II
code=GRU|0x200 precision=1                               | UU II II UU UU
code=GRU|0x200 precision=4                               | UU II II UU UU
code=LSTM|ACTIONS|0x200                                  | II II II II II
code=LSTM|ACTIONS|0x200 B=0                              | II II II II II
code=LSTM|ACTIONS|0x200 precision=1                      | UU II II UU UU
code=LSTM|ACTIONS|0x200 precision=4                      | UU II II UU UU
code=0x40000                                             | II II II II II
code=0x40000 B=0                                         | II II II II II
code=0x40000 precision=1                                 | UU II II UU UU
code=0x40000 precision=4                                 | UU II II UU UU
code=-1                                                  | II II II II II
code=-1 B=0                                              | II II II II II
code=-1 precision=1                                      | UU UU UU UU UU
code=-1 precision=4                                      | UU UU UU UU UU
n_layers=0                                               | II II II II II
n_layers=0 precision=1                                   | UU UU UU UU UU
n_layers=9                                               | II II II II II
n_layers=9 precision=1                                   | UU UU UU UU UU
n_layers=-1                                              | II II II II II
n_layers=-1 precision=1                                  | UU UU UU UU UU
"""

CELL_COLUMNS = ("cell", "sequence")
CELL_ROWS = """
n_layers=1                            | II II
n_layers=1 B=0                        | II II
n_layers=1 pairs=0                    | II II
n_layers=1 precision=1                | UU UU
n_layers=3                            | II II
n_layers=3 B=0                        | II II
n_layers=3 pairs=0                    | II II
n_layers=3 precision=1                | UU UU
dims=(0,8,2,3)                        | II II
dims=(0,8,2,3) B=0                    | II II
dims=(0,8,2,3) pairs=0                | II II
dims=(0,8,2,3) precision=1            | UU UU
dims=(4,0,2,3)                        | II II
dims=(4,0,2,3) B=0                    | II II
dims=(4,0,2,3) pairs=0                | II II
dims=(4,0,2,3) precision=1            | UU UU
dims=(4,8,0,3)                        | II II
dims=(4,8,0,3) B=0                    | II II
dims=(4,8,0,3) pairs=0                | II II
dims=(4,8,0,3) precision=1            | UU UU
dims=(65537,8,2,3)                    | II II
dims=(65537,8,2,3) B=0                | II II
dims=(65537,8,2,3) pairs=0            | II II
dims=(65537,8,2,3) precision=1        | UU UU
dims=(4,8193,2,3)                     | II II
dims=(4,8193,2,3) B=0                 | II II
dims=(4,8193,2,3) pairs=0             | II II
dims=(4,8193,2,3) precision=1         | UU UU
dims=(4,8,65537,3)                    | II II
dims=(4,8,65537,3) B=0                | II II
dims=(4,8,65537,3) pairs=0            | II II
dims=(4,8,65537,3) precision=1        | UU UU
dims=(65536,8192,65536,0)             | .. II
dims=(65536,8192,65536,0) B=0         | II II
dims=(65536,8192,65536,0) pairs=0     | .I II
dims=(65536,8192,65536,0) precision=1 | UU UU
dims=(4,8,2,0)                        | .. II
dims=(4,8,2,0) B=0                    | II II
dims=(4,8,2,0) pairs=0                | .I II
dims=(4,8,2,0) precision=1            | UU UU
dims=(4,8,2,-1)                       | .. II
dims=(4,8,2,-1) B=0                   | II II
dims=(4,8,2,-1) pairs=0               | .I II
dims=(4,8,2,-1) precision=1           | UU UU
"""

CNN_ROWS = """
code=N_CONV(1)|2                                                    | II
code=N_CONV(1)|2 B=0                                                | II
code=N_CONV(1)|2 precision=1                                        | UU
code=N_CONV(8)                                                      | II
code=N_CONV(8) B=0                                                  | II
code=N_CONV(8) precision=1                                          | UU
code=N_CONV(255)                                                    | II
code=N_CONV(255) B=0                                                | II
code=N_CONV(255) precision=1                                        | UU
code=N_CONV(1)|ACTIONS                                              | UU
code=N_CONV(1)|ACTIONS B=0                                          | UU
code=N_CONV(1)|ACTIONS precision=1                                  | UU
code=N_CONV(1)|GRU                                                  | UU
code=N_CONV(1)|GRU B=0                                              | UU
code=N_CONV(1)|GRU precision=1                                      | UU
code=N_CONV(1)|GRU|ACTIONS                                          | UU
code=N_CONV(1)|GRU|ACTIONS B=0                                      | UU
code=N_CONV(1)|GRU|ACTIONS precision=1                              | UU
code=N_CONV(8)|ACTIONS                                              | II
code=N_CONV(8)|ACTIONS B=0                                          | II
code=N_CONV(8)|ACTIONS precision=1                                  | UU
code=N_CONV(1)|ACTIONS theta=NULL                                   | UU
code=N_CONV(1)|ACTIONS ctx=NULL                                     | UU
code=N_CONV(1)|ACTIONS bc_plus=NULL bc_minus=FAKE                   | UU
code=N_CONV(8)|ACTIONS theta=NULL                                   | II
code=N_CONV(1)|XENT|OUT_TANH                                        | II
code=N_CONV(1)|XENT|OUT_TANH B=0                                    | II
code=N_CONV(1)|XENT|OUT_TANH precision=1                            | UU
code=N_CONV(1)|XENT|OUT_TANH|1                                      | II
code=N_CONV(1)|XENT|OUT_TANH|1 B=0                                  | II
code=N_CONV(1)|XENT|OUT_TANH|1 precision=1                          | UU
n_layers=1                                                          | II
n_layers=1 B=0                                                      | II
n_layers=1 centre_return_out=FAKE                                   | UU
n_layers=9                                                          | II
n_layers=9 B=0                                                      | II
n_layers=9 centre_return_out=FAKE                                   | UU
dims=(IN(0,8,8),CNN_CONV,4)                                         | II
dims=(IN(0,8,8),CNN_CONV,4) B=0                                     | II
dims=(IN(0,8,8),CNN_CONV,4) centre_return_out=FAKE                  | UU
dims=(IN(1,0,8),CNN_CONV,4)                                         | II
dims=(IN(1,0,8),CNN_CONV,4) B=0                                     | II
dims=(IN(1,0,8),CNN_CONV,4) centre_return_out=FAKE                  | UU
dims=(IN(1,8,0),CNN_CONV,4)                                         | II
dims=(IN(1,8,0),CNN_CONV,4) B=0                                     | II
dims=(IN(1,8,0),CNN_CONV,4) centre_return_out=FAKE                  | UU
dims=(CNN_IN|1<<30,CNN_CONV,4)                                      | II
dims=(CNN_IN|1<<30,CNN_CONV,4) B=0                                  | II
dims=(CNN_IN|1<<30,CNN_CONV,4) centre_return_out=FAKE               | UU
dims=(CNN_IN,CONV(0,3,1,0),4)                                       | II
dims=(CNN_IN,CONV(0,3,1,0),4) B=0                                   | II
dims=(CNN_IN,CONV(0,3,1,0),4) centre_return_out=FAKE                | UU
dims=(CNN_IN,CONV(2,0,1,0),4)                                       | II
dims=(CNN_IN,CONV(2,0,1,0),4) B=0                                   | II
dims=(CNN_IN,CONV(2,0,1,0),4) centre_return_out=FAKE                | UU
dims=(CNN_IN,CONV(2,3,0,0),4)                                       | II
dims=(CNN_IN,CONV(2,3,0,0),4) B=0                                   | II
dims=(CNN_IN,CONV(2,3,0,0),4) centre_return_out=FAKE                | UU
dims=(CNN_IN,CONV(2,3,1,3),4)                                       | II
dims=(CNN_IN,CONV(2,3,1,3),4) B=0                                   | II
dims=(CNN_IN,CONV(2,3,1,3),4) centre_return_out=FAKE                | UU
dims=(CNN_IN,CONV(2,9,1,0),4)                                       | II
dims=(CNN_IN,CONV(2,9,1,0),4) B=0                                   | II
dims=(CNN_IN,CONV(2,9,1,0),4) centre_return_out=FAKE                | UU
dims=(CNN_IN,CNN_CONV|1<<30,4)                                      | II
dims=(CNN_IN,CNN_CONV|1<<30,4) B=0                                  | II
dims=(CNN_IN,CNN_CONV|1<<30,4) centre_return_out=FAKE               | UU
dims=(CNN_IN,CNN_CONV,0)                                            | II
dims=(CNN_IN,CNN_CONV,0) B=0                                        | II
dims=(CNN_IN,CNN_CONV,0) centre_return_out=FAKE                     | UU
dims=(IN(1023,1023,1023),CONV(4095,1,1,0),4)                        | II
dims=(IN(1023,1023,1023),CONV(4095,1,1,0),4) B=0                    | II
dims=(IN(1023,1023,1023),CONV(4095,1,1,0),4) centre_return_out=FAKE | UU
"""

CONV_COLUMNS = ("vbn", "actions")
CONV_ROWS = """
precision=0 B=0                     | II II
precision=1 B=0                     | II UU
precision=1                         | .. UU
precision=2 B=0                     | II UU
precision=2                         | UU UU
precision=3 B=0                     | II UU
precision=3                         | UU UU
precision=4 B=0                     | II UU
precision=4                         | UU UU
precision=7 B=0                     | II UU
precision=7                         | UU UU
ctx=NULL                            | II II
theta=NULL                          | II II
table=NULL                          | .I ..
xref=NULL                           | II ..
obs=NULL                            | II ..
target=NULL                         | II ..
returns_plus=NULL                   | II II
returns_minus=NULL                  | .I .I
scratch=NULL                        | II II
n_actions=0                         | II II
n_actions=65                        | II II
n_actions=ACTIONS                   | II II
n_actions=ACTIONS|65                | II II
n_actions=ACTIONS|0x106             | II II
n_actions=XENT|6                    | II II
n_actions=-1                        | II II
ref_batch=1                         | II II
ref_batch=0                         | II II
B=0                                 | II II
B=-1                                | II II
pairs=0                             | II .I
pairs=-1                            | II .I
pairs=MAX_PAIRS+1                   | II .I
xref=ODD                            | II II
obs=ODD                             | II II
scratch=ODD                         | .. II
xref=NULL obs=NULL                  | II II
scratch_bytes=0                     | .. II
scratch_bytes=-1                    | .. II
ctx=NULL precision=1                | II UU
theta=NULL precision=1              | II UU
table=NULL precision=1              | .I UU
table16=NULL precision=1            | .I UU
order=NULL precision=1              | .. UU
xref=NULL precision=1               | II UU
obs=NULL precision=1                | II UU
target=NULL precision=1             | II UU
returns_plus=NULL precision=1       | II UU
returns_minus=NULL precision=1      | .I UU
scratch=NULL precision=1            | II UU
n_actions=0 precision=1             | II II
n_actions=65 precision=1            | II II
n_actions=ACTIONS precision=1       | UU UU
n_actions=ACTIONS|65 precision=1    | UU UU
n_actions=ACTIONS|0x106 precision=1 | UU UU
n_actions=XENT|6 precision=1        | II II
n_actions=-1 precision=1            | II II
ref_batch=1 precision=1             | II UU
ref_batch=0 precision=1             | II UU
B=0 precision=1                     | II UU
B=-1 precision=1                    | II UU
pairs=0 precision=1                 | II UU
pairs=-1 precision=1                | II UU
pairs=MAX_PAIRS+1 precision=1       | II UU
xref=ODD precision=1                | II UU
obs=ODD precision=1                 | II UU
theta=ODD precision=1               | II UU
scratch=ODD precision=1             | II UU
table16=ODD precision=1             | II UU
xref=NULL obs=NULL precision=1      | II UU
scratch_bytes=0 precision=1         | .. UU
scratch_bytes=-1 precision=1        | .. UU
ctx=NULL precision=2                | II UU
theta=NULL precision=2              | II UU
table=NULL precision=2              | UI UU
table16=NULL precision=2            | UU UU
order=NULL precision=2              | UU UU
xref=NULL precision=2               | II UU
obs=NULL precision=2                | II UU
target=NULL precision=2             | II UU
returns_plus=NULL precision=2       | II UU
returns_minus=NULL precision=2      | UI UU
scratch=NULL precision=2            | II UU
n_actions=0 precision=2             | II II
n_actions=65 precision=2            | II II
n_actions=ACTIONS precision=2       | UU UU
n_actions=ACTIONS|65 precision=2    | UU UU
n_actions=ACTIONS|0x106 precision=2 | UU UU
n_actions=XENT|6 precision=2        | II II
n_actions=-1 precision=2            | II II
ref_batch=1 precision=2             | II UU
ref_batch=0 precision=2             | II UU
B=0 precision=2                     | II UU
B=-1 precision=2                    | II UU
pairs=0 precision=2                 | II UU
pairs=-1 precision=2                | II UU
pairs=MAX_PAIRS+1 precision=2       | II UU
xref=ODD precision=2                | II UU
obs=ODD precision=2                 | II UU
theta=ODD precision=2               | UU UU
scratch=ODD precision=2             | UU UU
table16=ODD precision=2             | UU UU
xref=NULL obs=NULL precision=2      | II UU
scratch_bytes=0 precision=2         | UU UU
scratch_bytes=-1 precision=2        | UU UU
"""


def _rows(table, columns):
    """(id, column, centre, overrides, expected status) of every call of a table."""
    out = []
    for line in table.strip().splitlines():
        args, codes = line.rsplit("|", 1)
        over = {k: eval(v, dict(NAMES)) for k, v in (tok.split("=", 1) for tok in args.split())}
        for col, pair in zip(columns, codes.split()):
            for centre, ch in zip((True, False), pair):
                if ch != ".":
                    rid = f"{col}-{'centre' if centre else 'population'}-{args.strip().replace(' ', '-')}"
                    out.append((rid, col, centre, over, {"I": I, "U": U}[ch]))
    return out


def _mlp_cases():
    return _rows(MLP_ROWS, MLP_COLUMNS) + _rows(CELL_ROWS, CELL_COLUMNS) + _rows(CNN_ROWS, ("cnn",))


@pytest.mark.parametrize("rid,route,centre,over,want", _mlp_cases(), ids=[c[0] for c in _mlp_cases()])
def test_eval_mlp_status(rid, route, centre, over, want):
    assert _eval_mlp(route, centre, **over) == want, _lib().estk_last_error().decode()


@pytest.mark.parametrize("rid,kind,centre,over,want", _rows(CONV_ROWS, CONV_COLUMNS),
                         ids=[c[0] for c in _rows(CONV_ROWS, CONV_COLUMNS)])
def test_eval_conv_vbn_status(rid, kind, centre, over, want):
    assert _eval_conv_vbn(kind == "actions", centre, **over) == want, _lib().estk_last_error().decode()
