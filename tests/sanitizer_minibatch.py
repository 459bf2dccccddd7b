"""A small pass over the minibatch sampler (estk_sample_batch, estk_batch.cu) for compute-sanitizer (memcheck /
racecheck): unaligned 3-float rows from an offset allocation, a batch that straddles two epochs, rows gathered by a
whole CTA (3072 floats), and a 2^26 + 3-row dataset at g near 2^40.  Each pass is checked against the host
restatement batch_indices and the dataset's bytes, so that a sanitizer run is also a correctness run.

    compute-sanitizer --tool memcheck python tests/sanitizer_minibatch.py
    compute-sanitizer --tool racecheck python tests/sanitizer_minibatch.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from estorch_b200 import batch_indices  # noqa: E402
from estorch_b200.backend import CudaBackend  # noqa: E402

be = CudaBackend(torch.device("cuda", 0))
for name, n, b, row, trow, offset, g in (
        ("unaligned", 1000, 256, 3, 2, 1, 3),
        ("straddling", 1000, 256, 16, 4, 0, 17),
        ("wide rows", 600, 64, 3072, 10, 2, 9),
        ("large N", (1 << 26) + 3, 1000, 1, 1, 0, (1 << 40) - 3)):
    base = torch.arange(n * row + offset, dtype=torch.float32, device=be.device)
    obs = base[offset:].view(n, row)
    tgt = -torch.arange(n * trow, dtype=torch.float32, device=be.device).view(n, trow)
    dst, tdst, idx = be.alloc(b, row), be.alloc(b, trow), be.zeros(b, dtype=torch.int64)
    be.sample_batch(5, None, g, obs, dst, tgt, tdst, idx)
    want = torch.from_numpy(batch_indices(5, g, n, b)).to(be.device)
    assert torch.equal(idx, want), name
    assert torch.equal(dst, obs[want]) and torch.equal(tdst, tgt[want]), name
    torch.cuda.synchronize()
    print(f"{name}: N={n} B={b} row={row} g={g}: ok")
print("sanitizer_minibatch: all passes ok")
