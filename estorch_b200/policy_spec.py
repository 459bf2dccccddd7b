"""Recognise policies the device kernels can evaluate.

The reference accepts any ``nn.Module`` class as ``policy`` and runs it on the
host (estorch.py:136,142,195-202).  The fused evaluate kernel needs the
architecture, so the module is inspected once: a chain
``Linear -> act -> ... -> Linear [-> Tanh]`` with ``act`` ReLU, Tanh, ELU (alpha 1),
SiLU or LeakyReLU (slope 0.01), the same on every hidden layer, whose parameters are registered in forward order
(examples/cartpole_es.py:6-20, examples/nsra_es.py:52-67) becomes an ``MLPSpec``.
Anything else returns ``None`` and the engine uses the materialising path (rows
built on the device, rollout on the host).  The conv + VirtualBatchNorm policy of the
Atari example becomes a ``ConvVBNSpec``, and a recurrent policy (one GRUCell / LSTMCell
and one Linear head, ``forward(x, state=None) -> (y, new_state)``) an ``RNNSpec``, which
population mode steps.
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


_CELL_CODES = {"gru": 8, "lstm": 9}  # estk.h ESTK_CELL_GRU / ESTK_CELL_LSTM


@dataclass(frozen=True)
class RNNSpec:
    """A recurrent policy: one ``nn.GRUCell`` / ``nn.LSTMCell`` (in -> H, with biases), then one ``nn.Linear``
    head (H -> out, with bias), optionally a Tanh output; ``forward(x, state=None) -> (y, new_state)`` with
    ``state`` = h (GRU) or (h, c) (LSTM), None meaning zeros."""
    cell: str                   # "gru" or "lstm"
    dims: tuple                 # (in, H, out)
    output: str = "identity"    # "identity" or "tanh"

    @property
    def act(self) -> int:
        """The ``estk_mlp_desc.activation`` code without ESTK_ACTIONS (include/estk.h)."""
        return _CELL_CODES[self.cell] | _OUTPUT_CODES[self.output]

    @property
    def gates(self) -> int:
        return 3 if self.cell == "gru" else 4

    @property
    def state_width(self) -> int:
        """S: the floats of state per observation (h, and c for LSTM)."""
        return self.dims[1] * (1 if self.cell == "gru" else 2)

    @property
    def n_parameters(self) -> int:
        i, h, o = self.dims
        return self.gates * h * (i + h + 2) + o * (h + 1)


def _cell_step(cell, x, state, w_ih, w_hh, b_ih, b_hh):
    """torch's GRUCell / LSTMCell step from explicit parameters; ``state`` None = zeros."""
    H = w_hh.shape[1]
    if cell == "gru":
        h = torch.zeros(x.shape[0], H, dtype=x.dtype, device=x.device) if state is None else state
        a = torch.nn.functional.linear(x, w_ih, b_ih).chunk(3, 1)
        b = torch.nn.functional.linear(h, w_hh, b_hh).chunk(3, 1)
        r, z = torch.sigmoid(a[0] + b[0]), torch.sigmoid(a[1] + b[1])
        n = torch.tanh(a[2] + r * b[2])
        return (1 - z) * n + z * h
    h, c = (torch.zeros(x.shape[0], H, dtype=x.dtype, device=x.device),) * 2 if state is None else state
    g = (torch.nn.functional.linear(x, w_ih, b_ih) + torch.nn.functional.linear(h, w_hh, b_hh)).chunk(4, 1)
    c2 = torch.sigmoid(g[1]) * c + torch.sigmoid(g[0]) * torch.tanh(g[2])
    return torch.sigmoid(g[3]) * torch.tanh(c2), c2


def _max_rel_ok(y, want) -> bool:
    return (torch.is_tensor(y) and y.shape == want.shape and
            bool((y - want).abs().max() <= 1e-4 * want.abs().max() + 1e-5))


def rnn_spec_from_module(module: nn.Module) -> Optional[RNNSpec]:
    """Return the RNNSpec of ``module`` or None.

    Structural test: the leaf modules are exactly one ``nn.GRUCell`` / ``nn.LSTMCell`` with ``bias=True``,
    one ``nn.Linear`` with a bias whose input width is the cell's ``hidden_size``, and at most one
    ``nn.Tanh``; the parameters are registered in the order cell, head.  Behavioural test: with parameters
    redrawn at a scale that keeps every gate and output O(1), the module's ``forward(x, state)`` and
    ``forward(x, None)`` are compared with the cell step + head for an identity and a Tanh output; the
    module is accepted only when exactly one output matches both, and it matches under the module's own
    parameters too.  Only a private ``torch.Generator`` draws: the global RNG stream is not touched.
    Stacked cells, ``nn.GRU`` / ``nn.LSTM``, ``nn.RNNCell``, deeper heads, a Linear before the cell and a
    forward that ignores the state all return None."""
    leaves = _leaf_modules(module)
    cells = [m for m in leaves if type(m) in (nn.GRUCell, nn.LSTMCell)]
    linears = [m for m in leaves if type(m) is nn.Linear]
    tanhs = [m for m in leaves if type(m) is nn.Tanh]
    if len(cells) != 1 or len(linears) != 1 or len(tanhs) > 1 or len(leaves) != 2 + len(tanhs):
        return None
    cell, head = cells[0], linears[0]
    if not cell.bias or head.bias is None or head.in_features != cell.hidden_size:
        return None
    params = list(module.parameters())
    expect = [cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh, head.weight, head.bias]
    if len(params) != len(expect) or any(a is not b for a, b in zip(params, expect)):
        return None
    kind = "gru" if isinstance(cell, nn.GRUCell) else "lstm"
    I, H, O = cell.input_size, cell.hidden_size, head.out_features
    names = [n for n, _ in module.named_parameters()]
    dev, dt = params[0].device, params[0].dtype
    g = torch.Generator().manual_seed(0x5EED)
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=dt).to(dev)  # noqa: E731

    def states():
        return rnd(5, H) if kind == "gru" else (rnd(5, H), rnd(5, H))

    def want(x, state, ps, output):
        s = _cell_step(kind, x, state, *ps[:4])
        h = s if kind == "gru" else s[0]
        y = torch.nn.functional.linear(h, ps[4], ps[5])
        return (torch.tanh(y) if output == "tanh" else y), s

    def same(got, x, state, ps, output):
        if not (isinstance(got, tuple) and len(got) == 2):
            return False
        y, s = want(x, state, ps, output)
        if not _max_rel_ok(got[0], y):
            return False
        if kind == "gru":
            return _max_rel_ok(got[1], s)
        return (isinstance(got[1], tuple) and len(got[1]) == 2 and _max_rel_ok(got[1][0], s[0])
                and _max_rel_ok(got[1][1], s[1]))

    with torch.no_grad():
        redrawn = [rnd(cell.weight_ih.shape[0], I) / I ** 0.5, rnd(cell.weight_hh.shape[0], H) / H ** 0.5,
                   rnd(cell.weight_ih.shape[0]), rnd(cell.weight_ih.shape[0]), rnd(O, H) / H ** 0.5, rnd(O)]
        own = [p.detach() for p in params]
        xr, sr, x, s = rnd(5, I), states(), rnd(5, I), states()
        try:
            call = lambda ps, xx, ss: torch.func.functional_call(module, dict(zip(names, ps)), (xx, ss))  # noqa
            got_r, got_r0, got, got0 = call(redrawn, xr, sr), call(redrawn, xr, None), call(own, x, s), call(own, x, None)
        except Exception:
            return None
        hits = [o for o in ("identity", "tanh")
                if same(got_r, xr, sr, redrawn, o) and same(got_r0, xr, None, redrawn, o)]
        if len(hits) != 1 or not (same(got, x, s, own, hits[0]) and same(got0, x, None, own, hits[0])):
            return None
    return RNNSpec(kind, (I, H, O), hits[0])


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
        # max-norm relative, not element by element: over raw 0..255 reference frames that are constant at many
        # pixels, VBN scales by ~1/sqrt(1e-5) and the small outputs carry amplified fp32 order differences
        if y.shape != want.shape or not bool((y - want).abs().max() <= 1e-3 * want.abs().max() + 1e-4):
            return None
    return ConvVBNSpec(int(f2.out_features), int(xref.shape[0]))
