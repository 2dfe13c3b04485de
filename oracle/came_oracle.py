"""Plain-torch restatement of came_pytorch 0.1.3 `CAME.step` (the optimizer every PixArt-Sigma config selects as
`CAMEWrapper`, diffusion/utils/optimizer.py:242-246) and of `torch.nn.utils.clip_grad_norm_` (train_scripts/train.py:181-182).

A per-parameter loop, op for op in came_pytorch's order, that runs in whatever dtype / device the tensors have (fp32 or fp64,
CPU or GPU).  came_pytorch is not a dependency: the restatement follows the package's published source and is the reference
the tests hold the fused kernels (`optim.FlatCAME`, `optim.clip_grad_norm_`) to.  State keys are came_pytorch's.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch


def _rms(t: torch.Tensor) -> torch.Tensor:
    return t.norm(2) / (t.numel() ** 0.5)


def _approx_sq_grad(row: torch.Tensor, col: torch.Tensor) -> torch.Tensor:
    r_factor = (row / row.mean(dim=-1, keepdim=True)).rsqrt_().unsqueeze(-1)
    c_factor = col.unsqueeze(-2).rsqrt()
    return torch.mul(r_factor, c_factor)


def init_state(p: torch.Tensor) -> Dict[str, object]:
    shape = p.shape
    st: Dict[str, object] = {"step": 0, "exp_avg": torch.zeros_like(p)}
    if p.dim() >= 2:
        st["exp_avg_sq_row"] = torch.zeros(shape[:-1], dtype=p.dtype, device=p.device)
        st["exp_avg_sq_col"] = torch.zeros(shape[:-2] + shape[-1:], dtype=p.dtype, device=p.device)
        st["exp_avg_res_row"] = torch.zeros(shape[:-1], dtype=p.dtype, device=p.device)
        st["exp_avg_res_col"] = torch.zeros(shape[:-2] + shape[-1:], dtype=p.dtype, device=p.device)
    else:
        st["exp_avg_sq"] = torch.zeros_like(p)
    st["RMS"] = 0
    return st


@torch.no_grad()
def came_step(params: Sequence[torch.Tensor], grads: Sequence[Optional[torch.Tensor]], states: List[Dict[str, object]], *,
              lr: float = 2e-5, eps: Tuple[float, float] = (1e-30, 1e-16), clip_threshold: float = 1.0,
              betas: Tuple[float, float, float] = (0.9, 0.999, 0.9999), weight_decay: float = 0.0) -> None:
    """One CAME step, in place on `params` and `states` (a list of dicts, empty dicts are initialised).  A parameter whose
    gradient is None is skipped, as came_pytorch skips `p.grad is None`."""
    for p, grad, state in zip(params, grads, states):
        if grad is None:
            continue
        if not state:
            state.update(init_state(p))
        factored = grad.dim() >= 2
        state["step"] += 1
        state["RMS"] = _rms(p)
        update = (grad ** 2) + eps[0]
        if factored:
            row, col = state["exp_avg_sq_row"], state["exp_avg_sq_col"]
            row.mul_(betas[1]).add_(update.mean(dim=-1), alpha=1.0 - betas[1])
            col.mul_(betas[1]).add_(update.mean(dim=-2), alpha=1.0 - betas[1])
            update = _approx_sq_grad(row, col)
            update.mul_(grad)
        else:
            v = state["exp_avg_sq"]
            v.mul_(betas[1]).add_(update, alpha=1.0 - betas[1])
            update = v.rsqrt().mul_(grad)
        update.div_((_rms(update) / clip_threshold).clamp_(min=1.0))
        exp_avg = state["exp_avg"]
        exp_avg.mul_(betas[0]).add_(update, alpha=1 - betas[0])
        res = (update - exp_avg) ** 2 + eps[1]
        if factored:
            rrow, rcol = state["exp_avg_res_row"], state["exp_avg_res_col"]
            rrow.mul_(betas[2]).add_(res.mean(dim=-1), alpha=1.0 - betas[2])
            rcol.mul_(betas[2]).add_(res.mean(dim=-2), alpha=1.0 - betas[2])
            update = _approx_sq_grad(rrow, rcol).mul_(exp_avg)
        else:
            update = exp_avg.clone()
        if weight_decay != 0:
            p.add_(p, alpha=-weight_decay * lr)
        update.mul_(lr)
        p.add_(-update)


@torch.no_grad()
def clip_grad_norm(grads: Iterable[torch.Tensor], max_norm: float, grad_scale: float = 1.0) -> torch.Tensor:
    """`torch.nn.utils.clip_grad_norm_` semantics on gradient tensors, in place, after multiplying them by grad_scale:
    total = ||(||g_i||)_i||, g_i *= min(max_norm / (total + 1e-6), 1).  Returns total (0-d)."""
    grads = list(grads)
    if grad_scale != 1.0:
        for g in grads:
            g.mul_(grad_scale)
    total = torch.stack([g.norm(2) for g in grads]).norm(2)
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    for g in grads:
        g.mul_(coef)
    return total
