"""TEST-ONLY: the seeded dataset of the minibatch tests."""
import numpy as np
import torch


def dataset(n, din, dout, seed=0, classes=False):
    """A seeded regression (or one-hot classification) dataset of n rows: obs [n, din], target [n, dout]."""
    rng = np.random.RandomState(seed)
    x = rng.standard_normal((n, din)).astype(np.float32)
    if classes:
        y = np.eye(dout, dtype=np.float32)[rng.randint(0, dout, n)]
    else:
        y = (0.5 * np.tanh(x @ rng.standard_normal((din, dout)))).astype(np.float32)
    return torch.from_numpy(x), torch.from_numpy(y)
