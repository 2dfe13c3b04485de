"""Optimizer steps and gradient clipping on the flat gradient buckets (SURVEY.md 8f.3).

Two optimizers, one per model family, as the reference's configs choose them (built by `diffusion/utils/optimizer.py:236-246`):
- `FlatCAME` -- `CAMEWrapper(lr=2e-5, weight_decay=0.0, betas=(0.9, 0.999, 0.9999), eps=(1e-30, 1e-16))` (came_pytorch.CAME), the
  optimizer of every PixArt-Sigma config (configs/pixart_sigma_config/*).  One `pxa_came_flat` call = 7 launches per step over
  ALL buckets, driven by a parameter table uploaded once; 32 B of HBM traffic per parameter.
- `FlatAdamW` -- `AdamW(lr=1e-4, weight_decay=3e-2, eps=1e-10)`, the optimizer of the PixArt-alpha configs
  (`configs/PixArt_xl2_internal.py:48`): one `pxa_adamw_flat` launch per bucket (29 launches, 28 B of HBM traffic per
  parameter), torch.optim.AdamW's update rule exactly (decoupled weight decay, bias-corrected first / second moments),
  optionally with the gradient un-scaling of a loss scaler folded in.
torch's optimizers walk 437 parameter tensors; here the parameters of a bucket of `parallel.GradBucketReducer` are views of ONE
flat fp32 buffer, like their gradients.  `clip_grad_norm_` is `torch.nn.utils.clip_grad_norm_` (train_scripts/train.py:181-182)
over the same buckets, with the norm kept on the device.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

from . import lib
from .parallel import GradBucketReducer


class FlatAdamW:
    """AdamW over the buckets of a `GradBucketReducer` whose parameters have been flattened (`reducer.flatten_params()`)."""

    def __init__(self, reducer: GradBucketReducer, lr: float = 2e-5, betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-10,
                 weight_decay: float = 3e-2):
        self.reducer = reducer
        self.lr, self.betas, self.eps, self.weight_decay = lr, betas, eps, weight_decay
        self.step_count = 0
        reducer.flatten_params()
        self.state = [{"exp_avg": torch.zeros_like(b["flat_param"]), "exp_avg_sq": torch.zeros_like(b["flat_param"])}
                      for b in reducer.buckets]

    def zero_grad(self, set_to_none: bool = False) -> None:
        self.reducer.zero_grad()

    @torch.no_grad()
    def step(self, grad_scale: float = 1.0) -> None:
        """One update of every parameter from the (already all-reduced) flat gradients.  grad_scale: multiplied into the
        gradients first (1 / loss scale)."""
        self.step_count += 1
        self.reducer.check_views()
        for b, st in zip(self.reducer.buckets, self.state):
            if b["flat_param"].dtype != torch.float32:
                raise RuntimeError("FlatAdamW updates fp32 master parameters (use model.float())")
            lib.adamw_flat(b["flat_param"], b["flat"], st["exp_avg"], st["exp_avg_sq"], step=self.step_count, lr=self.lr,
                           betas=self.betas, eps=self.eps, weight_decay=self.weight_decay, grad_scale=grad_scale)

    def state_dict(self) -> dict:
        return {"step": self.step_count, "lr": self.lr, "betas": self.betas, "eps": self.eps, "weight_decay": self.weight_decay,
                "state": [{k: v.clone() for k, v in st.items()} for st in self.state]}

    def load_state_dict(self, sd: dict) -> None:
        self.step_count = int(sd["step"])
        for st, src in zip(self.state, sd["state"]):
            for k in st:
                st[k].copy_(src[k])


@torch.no_grad()
def clip_grad_norm_(reducer: GradBucketReducer, max_norm: float, grad_scale: float = 1.0) -> torch.Tensor:
    """`torch.nn.utils.clip_grad_norm_(params, max_norm)` over the gradient buckets of `reducer`, in place, in two launches
    (`pxa_grad_clip_flat`): gradients are first multiplied by `grad_scale` (1 / loss scale, folding an unscale step in), then
    total = their 2-norm and every gradient is multiplied by min(max_norm / (total + 1e-6), 1).  Returns total as a 0-d fp32
    device tensor; neither it nor the coefficient is read by the host, so the call neither syncs nor breaks CUDA-graph
    capture (the fp32 [1024] partial-sum workspace is allocated once per reducer, at the first call).  Works with
    `FlatAdamW` and `FlatCAME` alike.  The bucket padding is not touched."""
    reducer.check_views()
    flats = [b["flat"] for b in reducer.buckets]
    if any(not f.is_cuda or f.dtype != torch.float32 for f in flats):
        raise RuntimeError("clip_grad_norm_ clips fp32 gradient buckets on CUDA (use model.float().cuda())")
    ws = getattr(reducer, "_pxa_clip_partials", None)
    if ws is None or ws.device != flats[0].device:
        ws = torch.empty(lib.GRAD_CLIP_PARTS, dtype=torch.float32, device=flats[0].device)
        reducer._pxa_clip_partials = ws
    total = torch.empty((), dtype=torch.float32, device=flats[0].device)
    lib.grad_clip_flat(flats, ws, total, max_norm=max_norm, grad_scale=grad_scale,
                       lengths=[sum(p.numel() for p in b["params"]) for b in reducer.buckets])
    return total


def came_layout(reducer: GradBucketReducer) -> Tuple[List[Dict[str, int]], Dict[str, int]]:
    """The parameter table of `FlatCAME` without pointers: one entry per parameter, bucket by bucket, with its element offset
    in the bucket, numel, the matrix view (lead, R, C) of came_pytorch's factored statistics (ndim >= 2: lead = prod of the
    leading dimensions; 1-D: lead = R = 1, C = numel) and the offsets of its statistics in the shared state vectors.  Returns
    (entries, totals) with totals n_row / n_col / n_vec, the lengths of those vectors."""
    entries, n_row, n_col, n_vec = [], 0, 0, 0
    for bi, b in enumerate(reducer.buckets):
        off = 0
        for p in b["params"]:
            n = p.numel()
            e = dict(bucket=bi, offset=off, numel=n, bucket_numel=b["flat"].numel(), factored=int(p.dim() >= 2))
            if e["factored"]:
                e["R"], e["C"] = p.shape[-2], p.shape[-1]
                e["lead"] = n // (e["R"] * e["C"]) if n else 0
                e["sq_off"], e["col_off"] = n_row, n_col
                n_row += e["lead"] * e["R"]
                n_col += e["lead"] * e["C"]
            else:
                e.update(lead=1, R=1, C=n, sq_off=n_vec, col_off=0)
                n_vec += n
            entries.append(e)
            off += n
    return entries, dict(n_row=n_row, n_col=n_col, n_vec=n_vec)


class FlatCAME:
    """CAME (came_pytorch 0.1.3 `CAME.step`, selected as `CAMEWrapper` by every PixArt-Sigma config) over the buckets of a
    `GradBucketReducer` whose parameters are flattened here (`reducer.flatten_params()`).  Defaults: came_pytorch's
    constructor with the Sigma configs' lr.

    Every step updates every parameter of the reducer: in a bucket each parameter has a gradient view, zero if the parameter
    was unused, so -- unlike torch optimizers, which skip `p.grad is None` -- an unused parameter still gets a step (with a
    zero gradient).  State per parameter is came_pytorch's (exp_avg; factored row / column statistics of the second moment
    and of the instability for ndim >= 2, exp_avg_sq for 1-D; RMS of the parameter before the update), laid out flat:
    `to_torch_state_dict` / `load_torch_state_dict` convert it to / from the torch.optim checkpoint layout.

    `lr` lives in a device scalar, so an lr schedule can change it between replays of a CUDA graph that captured `step()`;
    the step itself never syncs or allocates."""

    def __init__(self, reducer: GradBucketReducer, lr: float = 2e-5, eps: Tuple[float, float] = (1e-30, 1e-16),
                 clip_threshold: float = 1.0, betas: Tuple[float, float, float] = (0.9, 0.999, 0.9999), weight_decay: float = 0.0):
        self.reducer = reducer
        self.eps, self.clip_threshold, self.betas, self.weight_decay = tuple(eps), clip_threshold, tuple(betas), weight_decay
        self.step_count = 0
        reducer.flatten_params()
        for b in reducer.buckets:
            if not b["flat_param"].is_cuda or b["flat_param"].dtype != torch.float32 or b["flat"].dtype != torch.float32:
                raise RuntimeError("FlatCAME updates fp32 master parameters on CUDA (use model.float().cuda())")
        dev = reducer.buckets[0]["flat_param"].device
        self.entries, totals = came_layout(reducer)
        self.exp_avg = [torch.zeros_like(b["flat_param"]) for b in reducer.buckets]
        z = lambda n: torch.zeros(max(n, 1), dtype=torch.float32, device=dev)
        self.exp_avg_sq, self.sq_row, self.res_row = z(totals["n_vec"]), z(totals["n_row"]), z(totals["n_row"])
        self.sq_col, self.res_col = z(totals["n_col"]), z(totals["n_col"])
        self.rms = z(len(self.entries))
        self._lr = torch.tensor([lr], dtype=torch.float32, device=dev)
        self._lr_host = float(lr)
        table = (lib.CameParam * len(self.entries))()
        for t, e in zip(table, self.entries):
            b = reducer.buckets[e["bucket"]]
            t.param = b["flat_param"].data_ptr() + 4 * e["offset"]
            t.grad = b["flat"].data_ptr() + 4 * e["offset"]
            t.exp_avg = self.exp_avg[e["bucket"]].data_ptr() + 4 * e["offset"]
            for k in ("numel", "offset", "bucket_numel", "sq_off", "col_off", "lead", "R", "C", "factored"):
                setattr(t, k, e[k])
        args = lib.CameArgs(exp_avg_sq=self.exp_avg_sq.data_ptr(), sq_row=self.sq_row.data_ptr(), res_row=self.res_row.data_ptr(),
                            sq_col=self.sq_col.data_ptr(), res_col=self.res_col.data_ptr(), rms=self.rms.data_ptr(),
                            lr=self._lr.data_ptr(), n_vec=totals["n_vec"], n_row=totals["n_row"], n_col=totals["n_col"],
                            eps1=self.eps[0], eps2=self.eps[1], clip_threshold=clip_threshold, beta1=self.betas[0],
                            beta2=self.betas[1], beta3=self.betas[2], weight_decay=weight_decay)
        nbytes = lib.came_plan(args, table)
        self.workspace = torch.empty(max(nbytes // 4, 4), dtype=torch.float32, device=dev)
        self.table = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8).to(dev)     # uploaded once
        args.table, args.workspace, args.workspace_bytes = self.table.data_ptr(), self.workspace.data_ptr(), self.workspace.numel() * 4
        self._args = args

    @property
    def lr(self) -> float:
        return self._lr_host

    @lr.setter
    def lr(self, value: float) -> None:
        """Written to the device scalar on the current stream (no sync): takes effect at the next step or graph replay."""
        self._lr_host = float(value)
        self._lr.fill_(self._lr_host)

    def state_bytes(self) -> int:
        """Bytes of optimizer state on the device (exp_avg, the factored / 1-D second moments, instability statistics)."""
        return sum(t.numel() * 4 for t in self.exp_avg + [self.exp_avg_sq, self.sq_row, self.res_row, self.sq_col, self.res_col])

    def zero_grad(self, set_to_none: bool = False) -> None:
        self.reducer.zero_grad()

    @torch.no_grad()
    def step(self) -> None:
        """One CAME update of every parameter from the (already all-reduced, optionally clipped) flat gradients."""
        self.step_count += 1
        self.reducer.check_views()
        self._args.step = self.step_count
        lib.came_flat(self._args)

    _STATE = ("exp_avg_sq", "sq_row", "res_row", "sq_col", "res_col", "rms")

    def state_dict(self) -> dict:
        return {"step": self.step_count, "lr": self.lr, "eps": self.eps, "clip_threshold": self.clip_threshold, "betas": self.betas,
                "weight_decay": self.weight_decay, "exp_avg": [t.clone() for t in self.exp_avg],
                **{k: getattr(self, k).clone() for k in self._STATE}}

    def load_state_dict(self, sd: dict) -> None:
        self.step_count = int(sd["step"])
        self.lr = sd["lr"]
        for dst, src in zip(self.exp_avg, sd["exp_avg"]):
            dst.copy_(src)
        for k in self._STATE:
            getattr(self, k).copy_(sd[k])

    # ------------------------------------------------------------------------------------------------ torch.optim layout
    def _views(self, e: Dict[str, int], p: torch.Tensor) -> Dict[str, torch.Tensor]:
        """came_pytorch's state tensors of one parameter, as views into the flat state."""
        o, n = e["offset"], e["numel"]
        out = {"exp_avg": self.exp_avg[e["bucket"]][o: o + n].view(p.shape)}
        if e["factored"]:
            lead_shape = p.shape[:-2]
            rows, cols = e["lead"] * e["R"], e["lead"] * e["C"]
            out["exp_avg_sq_row"] = self.sq_row[e["sq_off"]: e["sq_off"] + rows].view(*lead_shape, e["R"])
            out["exp_avg_sq_col"] = self.sq_col[e["col_off"]: e["col_off"] + cols].view(*lead_shape, e["C"])
            out["exp_avg_res_row"] = self.res_row[e["sq_off"]: e["sq_off"] + rows].view(*lead_shape, e["R"])
            out["exp_avg_res_col"] = self.res_col[e["col_off"]: e["col_off"] + cols].view(*lead_shape, e["C"])
        else:
            out["exp_avg_sq"] = self.exp_avg_sq[e["sq_off"]: e["sq_off"] + n].view(p.shape)
        return out

    def _entry_index(self) -> Dict[int, int]:
        idx, k = {}, 0
        for b in self.reducer.buckets:
            for p in b["params"]:
                idx[id(p)] = k
                k += 1
        return idx

    def to_torch_state_dict(self, model: torch.nn.Module) -> dict:
        """The state dict of the reference's `CAMEWrapper` as `train.py` checkpoints it (diffusion/utils/checkpoint.py): built
        by `MyOptimizerConstructor`, i.e. one param group per parameter in `model.parameters()` order, frozen parameters
        included (`requires_grad: False`, no state).  Per-parameter state: step, exp_avg, exp_avg_sq_row / _col,
        exp_avg_res_row / _col (ndim >= 2) or exp_avg_sq (1-D), RMS."""
        index = self._entry_index()
        state, groups = {}, []
        rms = self.rms.cpu()
        for k, p in enumerate(model.parameters()):
            g = {"lr": self.lr, "eps": self.eps, "clip_threshold": self.clip_threshold, "betas": self.betas,
                 "weight_decay": self.weight_decay}
            if not p.requires_grad:
                g["requires_grad"] = False
            g["params"] = [k]
            groups.append(g)
            if id(p) in index and self.step_count > 0:
                ei = index[id(p)]
                st = {"step": self.step_count}
                st.update({n: v.clone() for n, v in self._views(self.entries[ei], p).items()})
                st["RMS"] = rms[ei].clone().to(p.device)
                state[k] = st
        return {"state": state, "param_groups": groups}

    def load_torch_state_dict(self, model: torch.nn.Module, sd: dict) -> None:
        """Inverse of `to_torch_state_dict`: resume from a reference checkpoint's `optimizer` entry (or from this class's
        export).  The step count and lr are taken from the state / the param groups of the trainable parameters."""
        params = list(model.parameters())
        if len(sd["param_groups"]) != len(params):
            raise ValueError(f"expected one param group per model parameter ({len(params)}), got {len(sd['param_groups'])}")
        index = self._entry_index()
        steps, lrs = set(), set()
        with torch.no_grad():
            for k, (p, g) in enumerate(zip(params, sd["param_groups"])):
                if g["params"] != [k]:
                    raise ValueError(f"param group {k} holds {g['params']}, expected [{k}]")
                if id(p) not in index:
                    continue
                lrs.add(float(g["lr"]))
                st = sd["state"].get(k, sd["state"].get(str(k)))
                ei = index[id(p)]
                views = self._views(self.entries[ei], p)
                if st is None:                          # no step taken yet for this parameter
                    for v in views.values():
                        v.zero_()
                    self.rms[ei] = 0.0
                    continue
                for n, v in views.items():
                    v.copy_(st[n])
                self.rms[ei] = float(st["RMS"])
                steps.add(int(st["step"]))
        if len(steps) > 1:
            raise ValueError(f"parameters are at different steps {sorted(steps)}")
        self.step_count = steps.pop() if steps else 0
        if len(lrs) == 1:
            self.lr = lrs.pop()
