"""Recognise policies the device kernels can evaluate.

The reference accepts any ``nn.Module`` class as ``policy`` and runs it on the
host (estorch.py:136,142,195-202).  The fused evaluate kernel needs the
architecture, so the module is inspected once: a chain
``Linear -> act -> ... -> Linear [-> Tanh]`` with ``act`` ReLU, Tanh, ELU (alpha 1),
SiLU or LeakyReLU (slope 0.01), the same on every hidden layer, whose parameters are registered in forward order
(examples/cartpole_es.py:6-20, examples/nsra_es.py:52-67) becomes an ``MLPSpec``.
Anything else returns ``None`` and the engine uses the materialising path (rows
built on the device, rollout on the host).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch
from torch import nn


# estk.h ESTK_ACT_RELU / _TANH / _ELU / _SILU / _LEAKY_RELU
_HIDDEN_CODES = {"relu": 0, "tanh": 1, "elu": 3, "silu": 4, "leaky_relu": 5}
_OUTPUT_CODES = {"identity": 0, "tanh": 1 << 8}  # 0 / ESTK_ACT_OUT_TANH


@dataclass(frozen=True)
class MLPSpec:
    dims: tuple  # (in, h1, ..., out)
    hidden: str = "relu"        # activation after every Linear but the last: a key of _HIDDEN_CODES
    output: str = "identity"    # after the last Linear: "identity" or "tanh"

    @property
    def act(self) -> int:
        """The ``estk_mlp_desc.activation`` code of this policy (include/estk.h)."""
        return _HIDDEN_CODES[self.hidden] | _OUTPUT_CODES[self.output]

    @property
    def n_parameters(self) -> int:
        d = self.dims
        return sum(d[i] * d[i + 1] + d[i + 1] for i in range(len(d) - 1))


def _leaf_modules(module: nn.Module) -> List[nn.Module]:
    return [m for m in module.modules() if len(list(m.children())) == 0]


# the hidden kinds, their module types and the forms the kernels compute (default parameters only:
# estk_mlp_desc has no field for ELU's alpha or LeakyReLU's slope)
_F = torch.nn.functional
_HIDDEN = {"relu": (nn.ReLU, torch.relu), "tanh": (nn.Tanh, torch.tanh), "elu": (nn.ELU, _F.elu),
           "silu": (nn.SiLU, _F.silu), "leaky_relu": (nn.LeakyReLU, _F.leaky_relu)}


def _default_params(m: nn.Module) -> bool:
    if isinstance(m, nn.ELU):
        return float(m.alpha) == 1.0
    if isinstance(m, nn.LeakyReLU):
        return float(m.negative_slope) == 0.01
    return True


def _chain(x, linears, weights, hidden, output):
    h = x
    for i, (l, (w, b)) in enumerate(zip(linears, weights)):
        h = torch.nn.functional.linear(h, w, b)
        if i + 1 < len(linears):
            h = _HIDDEN[hidden][1](h)
    return torch.tanh(h) if output == "tanh" else h


def _matches(y, h) -> bool:
    return y.shape == h.shape and bool(torch.allclose(y, h, rtol=1e-4, atol=1e-5))


def mlp_spec_from_module(module: nn.Module, probe: bool = True) -> Optional[MLPSpec]:
    """Return the MLPSpec of ``module`` or None.

    Structural test: the leaf modules are only Linear / ReLU / Tanh / ELU / SiLU /
    LeakyReLU, ELU with ``alpha == 1`` and LeakyReLU with ``negative_slope == 0.01``;
    every Linear has a bias; widths chain; parameters are registered in layer order.
    Behavioural test (``probe``): a random batch through the module equals the
    chain evaluated from its flat parameters -- this rejects modules whose
    ``forward`` does something else with the same layers.

    The activations are found by the probe.  A hidden kind is a candidate if a leaf
    module of its type is registered, or if no activation module is (a ``forward``
    calling ``torch.relu`` / ``torch.tanh`` / ``F.elu`` / ``F.silu`` / ``F.leaky_relu``,
    every kind a candidate); the output is identity or,
    when Tanh is a candidate, Tanh.  Every (hidden, output) candidate pair is
    compared with the module's forward under parameters redrawn at a scale that
    keeps each layer's output O(1) (weights N(0, 1/fan_in), biases N(0, 1); the
    module's own parameters may be too small to tell ``tanh(y)`` from ``y``), and the
    module is accepted only when exactly one pair matches -- and matches under its
    own parameters too.  A single Linear has no hidden layer: its hidden kind is
    ``relu`` and only the output is probed.
    """
    leaves = _leaf_modules(module)
    linears = [m for m in leaves if isinstance(m, nn.Linear)]
    acts = tuple(t for t, _ in _HIDDEN.values())
    others = [m for m in leaves if not isinstance(m, (nn.Linear,) + acts) or not _default_params(m)]
    if not linears or others or len(linears) > 8:
        return None
    if any(l.bias is None for l in linears):
        return None
    dims = [linears[0].in_features]
    for l in linears:
        if l.in_features != dims[-1]:
            return None
        dims.append(l.out_features)
    params = list(module.parameters())
    expect = [p for l in linears for p in (l.weight, l.bias)]
    if len(params) != len(expect) or any(a is not b for a, b in zip(params, expect)):
        return None
    kinds = [k for k, (t, _) in _HIDDEN.items() if any(isinstance(m, t) for m in leaves)]
    kinds = kinds or list(_HIDDEN)
    hiddens = kinds if len(linears) > 1 else ["relu"]
    outputs = ["identity"] + (["tanh"] if "tanh" in kinds else [])
    cands = [(h, o) for h in hiddens for o in outputs]
    if not probe:                       # structure only: any activation but ReLU needs the probe to be placed
        return None if any(isinstance(m, acts) and not isinstance(m, nn.ReLU) for m in leaves) else MLPSpec(tuple(dims))
    with torch.no_grad():
        dev, dt = params[0].device, params[0].dtype
        # the same global-RNG draw as before Tanh was recognised: module initialisations that
        # follow the recognition (ES.__init__) see the same random stream
        x = torch.randn(3, dims[0], device=dev, dtype=dt)
        try:
            y = module(x)
        except Exception:
            return None
        own = [(l.weight, l.bias) for l in linears]
        # redrawn parameters from a private generator: the global RNG is not touched
        g = torch.Generator().manual_seed(0x5EED)
        xr = torch.randn(8, dims[0], generator=g, dtype=dt).to(dev)
        redrawn = [((torch.randn(l.out_features, l.in_features, generator=g, dtype=dt) / l.in_features ** 0.5).to(dev),
                    torch.randn(l.out_features, generator=g, dtype=dt).to(dev)) for l in linears]
        names = [n for n, _ in module.named_parameters()]
        try:
            yr = torch.func.functional_call(module, dict(zip(names, [t for wb in redrawn for t in wb])), (xr,))
        except Exception:
            return None
        hits = [c for c in cands if _matches(yr, _chain(xr, linears, redrawn, *c))]
        if len(hits) != 1 or not _matches(y, _chain(x, linears, own, *hits[0])):
            return None
    return MLPSpec(tuple(dims), *hits[0])


@dataclass(frozen=True)
class ConvVBNSpec:
    """The conv + VirtualBatchNorm policy of the reference's Atari example
    (examples/atari.py:14-37): conv1 4->16 k8 s4, VBN(16), conv2 16->32 k4 s2,
    VBN(32), fc1 2592->256, fc2 256->n_actions, with the reference batch ``xref``."""
    n_actions: int
    ref_batch: int

    @property
    def n_parameters(self) -> int:
        return 4096 + 16 + 16 + 16 + 8192 + 32 + 32 + 32 + 256 * 2592 + 256 + 256 * self.n_actions + self.n_actions


def conv_vbn_spec_from_module(module: nn.Module) -> Optional[ConvVBNSpec]:
    """Recognise the Atari-example architecture: leaf modules, in registration order,
    Conv2d(4,16,8,4) / VirtualBatchNorm(16) / Conv2d(16,32,4,2) / VirtualBatchNorm(32) /
    Linear(2592,256) / Linear(256,A), plus an ``xref`` tensor ``[R,4,84,84]``; the forward
    is probed against the same chain evaluated from the module's own parameters."""
    from .vbn import VirtualBatchNorm
    leaves = _leaf_modules(module)
    if len(leaves) != 6:
        return None
    c1, b1, c2, b2, f1, f2 = leaves
    ok = (isinstance(c1, nn.Conv2d) and (c1.in_channels, c1.out_channels, c1.kernel_size, c1.stride, c1.padding)
          == (4, 16, (8, 8), (4, 4), (0, 0)) and c1.bias is not None
          and isinstance(b1, VirtualBatchNorm) and b1.num_features == 16 and abs(b1.eps - 1e-5) < 1e-12
          and isinstance(c2, nn.Conv2d) and (c2.in_channels, c2.out_channels, c2.kernel_size, c2.stride, c2.padding)
          == (16, 32, (4, 4), (2, 2), (0, 0)) and c2.bias is not None
          and isinstance(b2, VirtualBatchNorm) and b2.num_features == 32 and abs(b2.eps - 1e-5) < 1e-12
          and isinstance(f1, nn.Linear) and (f1.in_features, f1.out_features) == (2592, 256) and f1.bias is not None
          and isinstance(f2, nn.Linear) and f2.in_features == 256 and f2.bias is not None)
    xref = getattr(module, "xref", None)
    if not ok or not torch.is_tensor(xref) or xref.dim() != 4 or tuple(xref.shape[1:]) != (4, 84, 84) or xref.shape[0] < 2:
        return None
    expect = [c1.weight, c1.bias, b1.weight, b1.bias, c2.weight, c2.bias, b2.weight, b2.bias,
              f1.weight, f1.bias, f2.weight, f2.bias]
    params = list(module.parameters())
    if len(params) != len(expect) or any(a is not b for a, b in zip(params, expect)):
        return None
    with torch.no_grad():
        F = torch.nn.functional
        dev = params[0].device
        x = torch.rand(2, 4, 84, 84, device=dev)
        xr = xref.to(dev)
        try:
            y = module(x)
        except Exception:
            return None

        def vbn(t, ref, m):
            mean, var = ref.mean(0, keepdim=True), ref.var(0, keepdim=True)
            return (t - mean) / torch.sqrt(var + m.eps) * m.weight.view(1, -1, 1, 1) + m.bias.view(1, -1, 1, 1)
        r1 = F.conv2d(xr, c1.weight, c1.bias, stride=4)
        h1 = torch.relu(vbn(F.conv2d(x, c1.weight, c1.bias, stride=4), r1, b1))
        r1n = torch.relu(vbn(r1, r1, b1))
        r2 = F.conv2d(r1n, c2.weight, c2.bias, stride=2)
        h2 = torch.relu(vbn(F.conv2d(h1, c2.weight, c2.bias, stride=2), r2, b2))
        want = F.linear(torch.relu(F.linear(h2.reshape(-1, 2592), f1.weight, f1.bias)), f2.weight, f2.bias)
        if y.shape != want.shape or not torch.allclose(y, want, rtol=1e-3, atol=1e-4):
            return None
    return ConvVBNSpec(int(f2.out_features), int(xref.shape[0]))
