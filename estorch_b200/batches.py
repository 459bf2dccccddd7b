"""Which dataset rows make up generation g's minibatch: the integer construction ``estk_sample_batch`` computes
on the device (include/estk_batch.h), restated on the host in numpy.  The two agree bit for bit, so a host rollout
(``DeviceAgent.set_generation``) sees exactly the batch the fused generation gathers."""
from __future__ import annotations

import numpy as np

_M64 = (1 << 64) - 1
_SALT = 0x6261746368657321          # the device's ESTK_BATCH_SALT
_ROUNDS = 4


def _mix64(z: int) -> int:
    """splitmix64 finaliser on a Python int (estk_mix64)."""
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def _mix64_np(z: np.ndarray) -> np.ndarray:
    """estk_mix64 element-wise on a uint64 array (numpy array arithmetic wraps modulo 2^64)."""
    z = z + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _half_bits(n: int) -> int:
    h = 1
    while (1 << (2 * h)) < n:
        h += 1
    return h


def _permute(r: np.ndarray, n: int, seed: int, epoch: int) -> np.ndarray:
    """pi_epoch(r) for a uint64 array r of values in [0, n)."""
    h = _half_bits(n)
    mask, sh = np.uint64((1 << h) - 1), np.uint64(h)
    ke = _mix64((_mix64((seed ^ _SALT) & _M64) + epoch) & _M64)
    keys = [np.uint64(_mix64((ke + k) & _M64)) for k in range(_ROUNDS)]
    x = r.astype(np.uint64)
    out = np.empty_like(x)
    todo = np.arange(x.size)
    while todo.size:                    # cycle walking: apply F again to the values that are still >= n
        L, R = x >> sh, x & mask
        for k in keys:
            L, R = R, L ^ (_mix64_np(k ^ R) & mask)
        x = (L << sh) | R
        done = x < np.uint64(n)
        out[todo[done]] = x[done]
        todo, x = todo[~done], x[~done]
    return out


def batch_indices(seed: int, generation: int, n_rows: int, batch: int) -> np.ndarray:
    """The ``batch`` dataset row indices (int64, in batch order) of minibatch ``generation`` of an ``n_rows``-row
    dataset under ``seed``: positions p = generation * batch + j of the stream of per-epoch permutations,
    row pi_e(p mod n_rows) with e = p div n_rows.  Every epoch visits every row once."""
    seed, g, n, b = int(seed) & _M64, int(generation), int(n_rows), int(batch)
    if not 0 < n < 1 << 31:
        raise ValueError(f"n_rows={n} outside [1, 2^31)")
    if not 0 < b <= n:
        raise ValueError(f"batch={b} outside [1, n_rows={n}]")
    if g < 0:
        raise ValueError(f"generation={g} is negative")
    e0, r0 = divmod(g * b, n)
    r = r0 + np.arange(b, dtype=np.int64)          # < 2n: epochs e0 and e0 + 1 at most
    nxt = r >= n
    out = np.empty(b, dtype=np.int64)
    out[~nxt] = _permute(r[~nxt], n, seed, e0).astype(np.int64)
    if nxt.any():
        out[nxt] = _permute(r[nxt] - n, n, seed, e0 + 1).astype(np.int64)
    return out
