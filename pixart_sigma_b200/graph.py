"""CUDA-graph replay of one denoiser forward (SURVEY.md 8f: removes ~310 kernel launches + their host work per step).

The C-ABI library never allocates or synchronises and the model forward has no host sync, so a whole
`PixArtMS.forward` captures into one CUDA graph.  `GraphedForward` keeps static input / output buffers per input
geometry, captures on first use (after two eager warm-up calls that size the workspace) and replays afterwards.
Small configurations (256 / 512 px) are launch-bound on the host without it; at 1024 px the GPU is the bottleneck
either way.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from .capture import capture_graph, kwargs_key, weights_key
from .lora import require_merged as require_lora_merged


class GraphedForward:
    """`method`: 'forward' or 'forward_with_dpmsolver' (the two entry points whose tensor arguments are x, timestep, y, mask;
    `forward_with_cfg` takes a guidance scale in that position and is not graphed here).  `data_info` tensors are captured
    by reference, so their identity is part of the graph key.  The returned tensor is a copy of the graph's static output."""

    METHODS = ("forward", "forward_with_dpmsolver")

    def __init__(self, model, method: str = "forward_with_dpmsolver"):
        if method not in self.METHODS:
            raise ValueError(f"GraphedForward supports {self.METHODS}, got {method!r}")
        self.model, self.method = model, method
        self._graphs: Dict[Tuple, dict] = {}
        self._wkey = None

    @torch.no_grad()
    def __call__(self, x: torch.Tensor, timestep: torch.Tensor, y: torch.Tensor, mask: Optional[torch.Tensor] = None,
                 data_info=None) -> torch.Tensor:
        require_lora_merged(self.model)           # a graph captured before an adapter was attached would ignore it
        dev = next(self.model.parameters()).device
        wkey = weights_key(self.model)                 # changes only when a replay could not see the parameters' update
        if wkey != self._wkey:
            self._graphs.clear()
            self._wkey = wkey
        key = (tuple(x.shape), tuple(y.shape), None if mask is None else tuple(mask.shape), kwargs_key(data_info))
        g = self._graphs.get(key)
        if g is None:
            st = {"x": torch.empty(x.shape, dtype=torch.float32, device=dev),
                  "t": torch.empty(timestep.shape, dtype=torch.float32, device=dev),
                  "y": torch.empty(y.shape, dtype=torch.bfloat16, device=dev),
                  "mask": None if mask is None else torch.empty(mask.shape, dtype=torch.long, device=dev)}
            self._copy_in(st, x, timestep, y, mask)
            fn = getattr(self.model, self.method)
            if self.method == "forward":
                call = lambda: fn(st["x"], st["t"], st["y"], mask=st["mask"], data_info=data_info)
            else:
                call = lambda: fn(st["x"], st["t"], st["y"], data_info=data_info, mask=st["mask"])
            # two eager warm-up calls: size the workspace, fill caches
            graph, out = capture_graph(lambda: (call(), call()), call, dev)
            g = {"graph": graph, "static": st, "out": out}
            self._graphs[key] = g
        self._copy_in(g["static"], x, timestep, y, mask)
        g["graph"].replay()
        return g["out"].clone()

    @staticmethod
    def _copy_in(st, x, t, y, mask):
        st["x"].copy_(x, non_blocking=True)
        st["t"].copy_(t, non_blocking=True)
        st["y"].copy_(y, non_blocking=True)
        if mask is not None:
            st["mask"].copy_(mask.reshape(st["mask"].shape), non_blocking=True)
