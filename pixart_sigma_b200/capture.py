"""What the native sampling loops share: the rule for when a captured CUDA graph may be replayed, the cache of captured loops,
the denoiser output as the step kernels read it, and the [uncond ; cond] batch of a guided call.

A captured loop reads its denoiser's parameters and every tensor in `model_kwargs` (nested ones included) by address, and
bakes scalars into its launches.  So a replay is valid only for the same callable, the same forward path (parameter dtype,
`output_dtype`), the same kwargs tensors at the same addresses and the same scalars; `denoiser_key` and the sampler's own
extras name all of them.
"""
from __future__ import annotations

import time
from typing import Callable, Dict, Optional

import torch

__all__ = ["CapturedLoops", "CfgCond", "capture_graph", "denoiser_key", "kwargs_key", "step_input", "weights_key"]


def kwargs_key(obj):
    """`obj` as a captured forward reads it: tensors by (address, shape, dtype, device), never by value (that would copy
    them to the host); dicts, lists and tuples element by element; anything else by value."""
    if isinstance(obj, torch.Tensor):
        return obj.data_ptr(), tuple(obj.shape), obj.dtype, obj.device
    if isinstance(obj, dict):
        return dict, tuple((k, kwargs_key(v)) for k, v in obj.items())
    if isinstance(obj, (list, tuple)):
        return type(obj), tuple(kwargs_key(v) for v in obj)
    return obj


def weights_key(owner) -> Optional[tuple]:
    """The parameters' part of a captured forward's key.  The kernels read the parameters in place, so a replay sees in-place
    updates by itself.  With `fuse_ln_modulate` the forward also keeps tables derived from them that a replay cannot refresh:
    then an in-place update (optimizer / EMA step) or a re-assignment (`.to(dtype)`) of a parameter changes the key."""
    if not getattr(owner, "fuse_ln_modulate", False):
        return None
    params = list(owner.parameters())
    return sum(p._version for p in params), params[0].data_ptr(), params[-1].data_ptr()


def denoiser_key(model: Callable, model_kwargs) -> tuple:
    """The denoiser's part of a captured loop's key: the module and function behind `model`, the parameter dtype and
    `output_dtype` (they select the forward's path), `model_kwargs` (`kwargs_key`) and the weights (`weights_key`)."""
    owner = getattr(model, "__self__", model)              # the nn.Module behind a bound forward_with_dpmsolver
    p = next(owner.parameters(), None) if isinstance(owner, torch.nn.Module) else None
    return (id(owner), getattr(model, "__func__", None), None if p is None else p.dtype, getattr(owner, "output_dtype", None),
            kwargs_key(model_kwargs), weights_key(owner))


def capture_graph(warmup: Callable[[], None], body: Callable, device=None):
    """Run `warmup` eagerly on a side stream (lazy inits, workspaces), then capture `body` into a CUDA graph.
    Returns (graph, what body returned)."""
    side = torch.cuda.Stream(device=device)
    side.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(side):
        warmup()
    torch.cuda.current_stream(device).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = body()
    return graph, out


class CapturedLoops:
    """The captured sampling loops of one sampler, by key; `len()` is the number captured."""

    def __init__(self):
        self._loops: Dict[tuple, tuple] = {}
        self.last_capture_s: Optional[float] = None          # wall time of the latest capture, warm-up included

    def __len__(self) -> int:
        return len(self._loops)

    def sample(self, model: Callable, model_kwargs, extras: tuple, x_T: torch.Tensor, draws, loop: Callable,
               keep: tuple = ()) -> torch.Tensor:
        """Replay the loop captured for this call, capturing it first if there is none, and return a copy of its output.

        extras: what else the loop bakes in or reads by address (plan scalars, guidance, `cond`'s address ...).
        draws: the per-step draws to replay, (steps, *x_T.shape) as a tensor or a sequence, or None when the loop draws.
        loop(x, k, draws): the sampler's loop from the latents x (left unchanged) over its first k steps (None: all) on
        `draws`; it allocates its own state (in the graph's memory pool when captured) and returns its output.
        keep: the other tensors the loop reads by address (`cond`, the timestep tensors), kept alive with the graph."""
        key = (denoiser_key(model, model_kwargs), tuple(x_T.shape), x_T.device, draws is None) + tuple(extras)
        entry = self._loops.get(key)
        if entry is None:
            x_in = torch.empty(x_T.shape, dtype=torch.float32, device=x_T.device)
            draws_in = None if draws is None else torch.zeros((len(draws),) + tuple(x_T.shape), device=x_T.device)
            zeros = torch.zeros((2,) + tuple(x_T.shape), device=x_T.device)
            t0 = time.perf_counter()
            # warm-up: the first two steps on zero draws, which consumes no random numbers
            graph, out = capture_graph(lambda: loop(x_T, 2, zeros), lambda: loop(x_in, None, draws_in))
            torch.cuda.synchronize(x_T.device)
            self.last_capture_s = time.perf_counter() - t0
            entry = self._loops[key] = (graph, x_in, draws_in, out, model, model_kwargs, keep)
        graph, x_in, draws_in, out = entry[:4]
        x_in.copy_(x_T)
        if isinstance(draws, torch.Tensor):
            draws_in.copy_(draws)
        elif draws is not None:
            for dst, src in zip(draws_in, draws):
                dst.copy_(src)
        graph.replay()
        return out.clone()


def step_input(out: torch.Tensor, fp16: bool = False) -> torch.Tensor:
    """The denoiser output as a step kernel reads it: fp32 or bf16 (and fp16 with `fp16`) with dense (h, w) planes (channel
    slices are fine)."""
    if out.dtype not in (torch.float32, torch.bfloat16) and not (fp16 and out.dtype == torch.float16):
        out = out.float()
    if not (out.stride(3) == 1 and out.stride(2) == out.shape[3] and out.stride(1) == out.shape[2] * out.shape[3]):
        out = out.contiguous()
    return out


class CfgCond:
    """[uncond ; cond] of a guided denoiser call, built once per input pair and rebuilt when either input changes, so that a
    captured loop reading it can be replayed."""

    def __init__(self):
        self._key, self._cat = None, None

    def __call__(self, uncond: torch.Tensor, cond: torch.Tensor) -> torch.Tensor:
        key = tuple((t.data_ptr(), t._version, tuple(t.shape), t.dtype) for t in (uncond, cond))
        if key != self._key:
            self._key, self._cat = key, torch.cat([uncond, cond])
        return self._cat
