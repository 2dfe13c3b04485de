"""LoRA on the functional PixArt-Sigma oracle (`pixart_oracle.forward` / `forward_grad`), on the CPU in fp32 or fp64.

Every adapted projection gets peft's LoRA layer on top of its base op:
    Linear  base(x) + lora_B(lora_A(x)) * scaling                          lora_A: Linear(K, r), lora_B: Linear(r, N), no bias
    Conv    base(x) + lora_B(lora_A(x)) * scaling                          lora_A: Conv2d(in, r, k, stride), lora_B: Conv2d(r, out, 1)
A fused native projection (attn.qkv: to_q / to_k / to_v; cross_attn.kv_linear: to_k / to_v) carries one such layer per
diffusers projection, each on its own slice of the output.  Adapters are given in the native layout of `lora.py`:
{native module name: (A [G r, ...], B [G, N / G, r])}; gradients come from torch autograd through `forward_grad`.

This restates peft's `LoraLayer.forward` for the configuration `train_pixart_lora_hf.py` uses (no dropout, no bias, no
DoRA).  peft and diffusers are not installed here, so the restatement is not pinned against peft itself.
"""
from __future__ import annotations

import contextlib
from typing import Dict, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import pixart_oracle as po

Adapters = Dict[str, Tuple[Tensor, Tensor]]


def lora_linear(x: Tensor, A: Tensor, B: Tensor, scaling: float) -> Tensor:
    """The adapter's contribution to a (fused) Linear: per group g, lora_B_g(lora_A_g(x)) * scaling on its output slice."""
    G, _, r = B.shape
    return torch.cat([F.linear(F.linear(x, A[g * r:(g + 1) * r]), B[g]) * scaling for g in range(G)], -1)


def lora_conv(x: Tensor, A: Tensor, B: Tensor, scaling: float, stride) -> Tensor:
    """peft's Conv2d LoRA: lora_A = Conv2d(in, r, k, stride), lora_B = 1x1 Conv2d(r, out)."""
    return F.conv2d(F.conv2d(x, A, stride=stride), B[0][:, :, None, None]) * scaling


class _Functional:
    """torch.nn.functional with the adapter of the patch-embedding convolution added to its conv2d."""

    def __init__(self, sd, adapters: Adapters, scaling: float):
        self._sd, self._ad, self._s = sd, adapters, scaling

    def __getattr__(self, name):
        return getattr(F, name)

    def conv2d(self, x, weight, bias=None, stride=1, *args, **kwargs):
        out = F.conv2d(x, weight, bias, stride, *args, **kwargs)
        ad = self._ad.get("x_embedder.proj")
        if ad is not None and weight is self._sd["x_embedder.proj.weight"]:
            out = out + lora_conv(x, ad[0], ad[1], self._s, stride)
        return out


@contextlib.contextmanager
def _with_adapters(sd, adapters: Adapters, scaling: float):
    lin, fn = po._lin, po.F

    def _lin(sd_, name, x):
        out = lin(sd_, name, x)
        ad = adapters.get(name)
        return out if ad is None else out + lora_linear(x, ad[0], ad[1], scaling)

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
    """`pixart_oracle.forward_grad` with the adapters applied unmerged: gradients reach the adapter tensors that require grad."""
    with _with_adapters(sd, adapters, scaling):
        return po.forward_grad(sd, cfg, x, timestep, y, mask=mask, data_info=data_info, dtype=dtype)


def merged_state_dict(sd, adapters: Adapters, scaling: float) -> Dict[str, Tensor]:
    """sd with W + scaling * blockdiag(B) A for every adapted projection (the merged weights)."""
    out = dict(sd)
    for name, (A, B) in adapters.items():
        G, _, r = B.shape
        w = sd[name + ".weight"]
        d = torch.cat([B[g] @ A[g * r:(g + 1) * r].flatten(1) for g in range(G)], 0)
        out[name + ".weight"] = w + scaling * d.view(w.shape)
    return out
