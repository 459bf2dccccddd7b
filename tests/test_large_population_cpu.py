"""The population limit: the Python binding agrees with include/estk.h, and ES refuses a population
beyond it at construction instead of in its first generation."""
import os
import re

import pytest
import torch

from conftest import ROOT
from _oracle_backend import OracleBackend
from test_api_cpu import MLP


def test_binding_limit_matches_header():
    from estorch_b200 import _capi
    text = open(os.path.join(ROOT, "include", "estk.h")).read()
    m = re.search(r"#define ESTK_MAX_POPULATION \(1 << (\d+)\)", text)
    assert m is not None
    assert _capi.ESTK_MAX_POPULATION == 1 << int(m.group(1)) == 1 << 22


def test_es_refuses_population_beyond_the_limit():
    import estorch_b200 as E
    obs, tgt = torch.zeros(8, 4), torch.zeros(8, 2)
    kw = dict(policy_kwargs={"dims": [4, 8, 2]}, agent_kwargs=dict(obs=obs, target=tgt),
              optimizer_kwargs={"lr": 0.01}, noise_table_size=1 << 12)
    with pytest.raises(ValueError, match="exceeds"):
        E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=(1 << 22) + 2, sigma=0.1,
             _backend=OracleBackend(), **kw)
    es = E.ES(MLP, E.DeviceAgent, torch.optim.Adam, population_size=1 << 16, sigma=0.1, _backend=OracleBackend(), **kw)
    assert es.population_size == 1 << 16
