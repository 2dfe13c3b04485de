"""DoRA on the functional PixArt-Sigma oracle, on the CPU in fp32 or fp64: `oracle/lora_oracle.py`'s peft LoRA layers with an
optional trained magnitude per adapter.

Adapters are {native module name: (A [G r, ...], B [G, N / G, r], m)} with m the fp32 magnitude [N] (concatenated over the
fused projections, as `lora_magnitude` on the native module) or None for a plain LoRA adapter.  With s the scaling,
    wn[n] = || W[n, :] + s (B A)[n, :] ||_2      per output row (over (in, kh, kw) for the conv), DETACHED (DoRA paper, 4.3)
    c     = m / wn
    y     = base(x) + (c - 1) (x W^T) + c s lora_B(lora_A(x))      (base(x) includes the bias, which c does not scale)
which is peft's DoRA layer for the reference script's configuration (no dropout, no bias) restated; peft is not installed
here, so the restatement is not pinned against peft itself.  Gradients come from torch autograd through `forward_grad`; the
norm is computed under no_grad, so no gradient flows through it.
"""
from __future__ import annotations

import contextlib
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import lora_oracle as lo
from oracle import pixart_oracle as po

Adapters = Dict[str, Tuple[Tensor, Tensor, Optional[Tensor]]]


def delta(w: Tensor, A: Tensor, B: Tensor, scaling: float) -> Tensor:
    """scaling * blockdiag(B) A, shaped like w."""
    G, _, r = B.shape
    return scaling * torch.cat([B[g] @ A[g * r:(g + 1) * r].flatten(1) for g in range(G)], 0).view(w.shape)


def col_scale(w: Tensor, A: Tensor, B: Tensor, m: Tensor, scaling: float) -> Tensor:
    """c = m / ||W + s B A||_row [N], the norm detached."""
    with torch.no_grad():
        wn = (w + delta(w, A, B, scaling)).flatten(1).norm(dim=1)
    return m / wn


def dora_linear(x: Tensor, w: Tensor, bias: Optional[Tensor], A: Tensor, B: Tensor, m: Optional[Tensor], scaling: float) -> Tensor:
    out = F.linear(x, w, bias)
    lora = lo.lora_linear(x, A, B, scaling)
    if m is None:
        return out + lora
    c = col_scale(w, A, B, m, scaling)
    return out + (c - 1) * F.linear(x, w) + c * lora


def dora_conv(x: Tensor, w: Tensor, bias: Optional[Tensor], A: Tensor, B: Tensor, m: Optional[Tensor], scaling: float,
              stride) -> Tensor:
    out = F.conv2d(x, w, bias, stride)
    lora = lo.lora_conv(x, A, B, scaling, stride)
    if m is None:
        return out + lora
    c = col_scale(w, A, B, m, scaling).view(1, -1, 1, 1)          # peft's conv magnitude layout [1, out, 1, 1]
    return out + (c - 1) * F.conv2d(x, w, None, stride) + c * lora


class _Functional:
    """torch.nn.functional with the adapter of the patch-embedding convolution applied to its conv2d."""

    def __init__(self, sd, adapters: Adapters, scaling: float):
        self._sd, self._ad, self._s = sd, adapters, scaling

    def __getattr__(self, name):
        return getattr(F, name)

    def conv2d(self, x, weight, bias=None, stride=1, *args, **kwargs):
        ad = self._ad.get("x_embedder.proj")
        if ad is not None and weight is self._sd["x_embedder.proj.weight"] and not args and not kwargs:
            return dora_conv(x, weight, bias, *ad, self._s, stride)
        return F.conv2d(x, weight, bias, stride, *args, **kwargs)


@contextlib.contextmanager
def _with_adapters(sd, adapters: Adapters, scaling: float):
    lin, fn = po._lin, po.F

    def _lin(sd_, name, x):
        ad = adapters.get(name)
        if ad is None:
            return lin(sd_, name, x)
        return dora_linear(x, sd_[name + ".weight"], sd_.get(name + ".bias"), *ad, scaling)

    po._lin, po.F = _lin, _Functional(sd, adapters, scaling)
    try:
        yield
    finally:
        po._lin, po.F = lin, fn


def forward(sd, adapters: Adapters, scaling: float, cfg, x, timestep, y, mask=None, data_info=None, dtype=torch.float32):
    """`pixart_oracle.forward` (no_grad) with the adapters applied unmerged."""
    with _with_adapters(sd, adapters, scaling):
        return po.forward(sd, cfg, x, timestep, y, mask=mask, data_info=data_info, dtype=dtype)


def forward_grad(sd, adapters: Adapters, scaling: float, cfg, x, timestep, y, mask=None, data_info=None, dtype=torch.float32):
    """`pixart_oracle.forward_grad` with the adapters applied unmerged: gradients reach A, B and m where they require grad."""
    with _with_adapters(sd, adapters, scaling):
        return po.forward_grad(sd, cfg, x, timestep, y, mask=mask, data_info=data_info, dtype=dtype)


def merged_state_dict(sd, adapters: Adapters, scaling: float) -> Dict[str, Tensor]:
    """sd with the merged weights: W + s blockdiag(B) A, and for DoRA c (W + s blockdiag(B) A) with c = m / ||W + s B A||_row."""
    out = dict(sd)
    for name, (A, B, m) in adapters.items():
        w = sd[name + ".weight"]
        new = w + delta(w, A, B, scaling)
        if m is not None:
            new = col_scale(w, A, B, m, scaling).view((-1,) + (1,) * (w.dim() - 1)) * new
        out[name + ".weight"] = new
    return out
