"""The noise-table length limit, without a GPU: estk_make_offsets and ES refuse a table longer than
ESTK_MAX_TABLE_LEN before they touch the device.

estk_make_offsets checks its arguments before it reads the context, so a fake non-null pointer stands in for the
context and the output buffers (none is dereferenced)."""
import ctypes as C
import os
import re

import pytest
import torch

from estorch_b200 import _capi
from conftest import ROOT

I = -1                            # ESTK_ERR_INVALID
FAKE = C.c_void_p(256)            # 16-byte aligned, never dereferenced
MAX = _capi.ESTK_MAX_TABLE_LEN


def _lib():
    if not os.path.exists(_capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _capi.load()


def test_header_and_binding_state_the_same_limit():
    text = open(os.path.join(ROOT, "include", "estk.h")).read()
    m = re.search(r"#define ESTK_MAX_TABLE_LEN \(1ll << (\d+)\)", text)
    assert m and MAX == 1 << int(m.group(1)) == 1 << 34


def _make_offsets(table_len, n=4610, pairs=4, order=True):
    return _lib().estk_make_offsets(FAKE, 1, None, 0, 0, pairs, table_len, n, FAKE, FAKE if order else None, None)


@pytest.mark.parametrize("table_len", [MAX + 32, MAX + 1, 2 * MAX, 1 << 40, (1 << 62) + 32])
@pytest.mark.parametrize("order", [True, False])
def test_make_offsets_refuses_a_table_beyond_the_limit(table_len, order):
    assert _make_offsets(table_len, order=order) == I
    msg = _lib().estk_last_error().decode()
    assert "estk_make_offsets" in msg and str(MAX) in msg and str(table_len) in msg


def test_make_offsets_still_refuses_a_table_shorter_than_a_row():
    assert _make_offsets(4096, n=4097) == I
    assert "padded row" in _lib().estk_last_error().decode()


class _Untouchable:
    """A backend stand-in that fails on any use: the refusal must come before the engine touches one."""

    def __getattr__(self, name):
        raise AssertionError(f"the backend was used ({name}) before the table length was checked")


@pytest.mark.parametrize("size", [MAX + 1, MAX + 32, 1 << 50])
def test_es_refuses_a_noise_table_beyond_the_limit(size):
    import estorch_b200 as E
    from test_api_cpu import MLP
    obs, tgt = torch.randn(8, 4), torch.randn(8, 2)
    with pytest.raises(ValueError, match=f"noise_table_size {size} exceeds .*{MAX} entries"):
        E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=8, sigma=0.02, policy_kwargs={"dims": [4, 8, 2]},
             agent_kwargs=dict(obs=obs, target=tgt), noise_table_size=size, _backend=_Untouchable())
