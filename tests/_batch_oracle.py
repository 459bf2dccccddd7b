"""TEST-ONLY: ``sample_batch`` (CudaBackend's signature) for the oracle stand-in backends, computed by the host
restatement ``batch_indices``, so the minibatch host logic runs without a GPU.  ``with_batches(cls)`` adds it to
any stand-in backend class (the MLP, CNN and sequence ones); ``BatchOracleBackend`` is the plain MLP one."""
import numpy as np
import torch

from estorch_b200.backend import STATE_DTYPE
from estorch_b200.batches import batch_indices
from _oracle_backend import OracleBackend


class BatchMixin:
    def sample_batch(self, seed, state, gen_host, obs_src, obs_dst, tgt_src, tgt_dst, index_out=None):
        g = gen_host + (int(state.numpy().view(STATE_DTYPE)["generation"][0]) if state is not None else 0)
        idx = torch.from_numpy(batch_indices(seed, g, obs_src.shape[0], obs_dst.shape[0]))
        obs_dst.copy_(obs_src[idx])
        tgt_dst.copy_(tgt_src[idx])
        if index_out is not None:
            index_out.copy_(idx)
        self.batch_calls = getattr(self, "batch_calls", 0) + 1
        self.launches += 1


def with_batches(cls):
    return type(cls.__name__ + "WithBatches", (BatchMixin, cls), {})


BatchOracleBackend = with_batches(OracleBackend)


def dataset(n, din, dout, seed=0, classes=False):
    """A seeded regression (or one-hot classification) dataset of n rows: obs [n, din], target [n, dout]."""
    rng = np.random.RandomState(seed)
    x = rng.standard_normal((n, din)).astype(np.float32)
    if classes:
        y = np.eye(dout, dtype=np.float32)[rng.randint(0, dout, n)]
    else:
        y = (0.5 * np.tanh(x @ rng.standard_normal((din, dout)))).astype(np.float32)
    return torch.from_numpy(x), torch.from_numpy(y)
