"""A small pass over the convolutional evaluate (estk_eval_cnn.cu) for compute-sanitizer (memcheck / racecheck /
synccheck): the shared-memory form on a four-conv shape with B = 257 (a tail chunk, several chunks per pair, the
last-arrival reduction), its centre form, and the slab form on a 3x128x128, 32-channel shape (a persistent grid
reusing per-CTA global buffers), each checked against the float64 forward so that a sanitizer run is also a
correctness run.

    compute-sanitizer --tool memcheck python tests/sanitizer_cnn.py
    compute-sanitizer --tool racecheck python tests/sanitizer_cnn.py
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from estorch_b200.backend import CudaBackend  # noqa: E402
from _cnn_oracle import pack  # noqa: E402
from test_cnn_gpu import SIGMA, TANH, XENT, _data, _eval, _forward64, _rel, _returns64, _setup  # noqa: E402

be = CudaBackend(torch.device("cuda", 0))
for shape, convs, linears, B, pairs, code in (
        ((2, 13, 13), [(3, 3, 2, 2), (7, 3, 1, 0), (5, 1, 1, 0), (4, 3, 1, 1)], [9, 6, 2], 257, 3, 3 | XENT | 4 << 24),
        ((3, 128, 128), [(32, 3, 1, 1), (4, 8, 8, 0)], [4], 2, 2, 1 | TANH | 2 << 24)):
    dims = pack(shape, convs, linears)
    theta, table, offsets, order = _setup(be, dims, code, pairs)
    obs, tgt = (t.to(be.device) for t in _data(shape, B, linears[-1], bool(code & XENT)))
    ret, y = _eval(be, dims, code, theta, table, offsets, order, pairs, SIGMA, obs, tgt)
    rows = be.alloc(2 * pairs, theta.numel())
    be.perturb_rows(theta, table, offsets, pairs, SIGMA, 0, 2 * pairs, rows)
    y64 = _forward64(rows, dims, code, obs)
    r64 = _returns64(y64, tgt, bool(code & XENT))
    assert _rel(y, y64) < 1e-5 and _rel(ret, r64) < 1e-5, (shape, _rel(y, y64), _rel(ret, r64))
    one, bc = be.zeros(1), be.zeros(B * linears[-1])
    be.eval_cnn_center(dims, theta, obs, tgt, one, bc, B, B * linears[-1], act=code)
    c64 = _forward64(theta[None], dims, code, obs)
    assert _rel(bc.view(1, B, -1), c64) < 1e-5 and _rel(one, _returns64(c64, tgt, bool(code & XENT))) < 1e-5
    torch.cuda.synchronize()
    print(f"{shape} B={B} pairs={pairs} code={code:#x}: ok")
print("sanitizer_cnn: all passes ok")
