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
        self._params = list(model.parameters())
        self._wkey = None

    @staticmethod
    def _key(x, y, mask, data_info):
        di = None
        if data_info is not None:
            di = tuple(sorted((k, (v.data_ptr(), tuple(v.shape)) if isinstance(v, torch.Tensor) else repr(v))
                              for k, v in data_info.items()))
        return (tuple(x.shape), tuple(y.shape), None if mask is None else tuple(mask.shape), di)

    @torch.no_grad()
    def __call__(self, x: torch.Tensor, timestep: torch.Tensor, y: torch.Tensor, mask: Optional[torch.Tensor] = None,
                 data_info=None) -> torch.Tensor:
        require_lora_merged(self.model)           # a graph captured before an adapter was attached would ignore it
        dev = self._params[0].device
        # The kernels read the parameters in place, but the fused-LN forward also keeps tables derived from them
        # that a captured graph cannot refresh: an in-place update or a re-assignment of any parameter (optimizer / EMA step,
        # .to(dtype)) drops the captured graphs.
        # (Without such copies -- the default configuration -- a replay reads the updated parameters in place and nothing is dropped.)
        wkey = (sum(p._version for p in self._params), self._params[0].data_ptr(), self._params[-1].data_ptr())
        if wkey != self._wkey:
            derived = getattr(self.model, "_ln_fusion", None) is not None
            if self._wkey is not None and derived:
                self._graphs.clear()
            self._wkey = wkey
        key = self._key(x, y, mask, data_info)
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
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for _ in range(2):                      # eager warm-up: sizes the workspace, fills caches
                    call()
            torch.cuda.current_stream(dev).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = call()
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
