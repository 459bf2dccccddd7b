"""A small pass over the TF32 convolutional evaluate (estk_eval_cnn_tf32.cu) for compute-sanitizer (memcheck /
racecheck / synccheck): a four-conv shape with B = 257 (three chunks per pair, a tail chunk, the last-arrival
reduction), its centre form, and a 3x128x128, 32-channel shape (one image per chunk, a persistent grid reusing
per-CTA slabs), each checked against the TF32 rounding model and the float64 forward so that a sanitizer run is
also a correctness run.

    compute-sanitizer --tool memcheck python tests/sanitizer_cnn_tf32.py
    compute-sanitizer --tool racecheck python tests/sanitizer_cnn_tf32.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from estorch_b200.backend import CudaBackend  # noqa: E402
from _cnn_oracle import forward, pack  # noqa: E402
from _cnn_tf32_oracle import forward_tf32  # noqa: E402
from test_cnn_tf32_gpu import BAR_MODEL, SIGMA, TANH, U, XENT, _data, _eval, _rel, _setup  # noqa: E402

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
    R, X = rows.cpu().numpy(), obs.cpu().numpy()
    e_model = _rel(y.cpu().numpy(), np.stack([forward_tf32(r, dims, code, X) for r in R]))
    e_64 = _rel(y.cpu().numpy(), np.stack([forward(r, dims, code, X, dt=np.float64) for r in R]))
    bar64 = 2 * (len(convs) + len(linears)) * U
    assert e_model <= BAR_MODEL and e_64 <= bar64, (e_model, e_64)
    rc, bc = be.zeros(1), be.zeros(B * linears[-1])
    be.eval_cnn_center(dims, theta, obs, tgt, rc, bc, B, B * linears[-1], precision="tf32", act=code)
    torch.cuda.synchronize()
    e_c = _rel(bc.cpu().numpy(), forward_tf32(theta.cpu().numpy(), dims, code, X).reshape(-1))
    assert e_c <= BAR_MODEL, e_c
    print(f"{shape} B={B}: outputs vs model {e_model:.2e}, vs float64 {e_64:.2e}, centre vs model {e_c:.2e}")
print("sanitizer_cnn_tf32 ok")
