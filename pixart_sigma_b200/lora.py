"""LoRA adapters on the native PixArtMS, in peft's directory format, with merged-weight sampling.

A LoRA adapter adds s * B A to a frozen linear weight W [N, K]: A [r, K], B [N, r], s = lora_alpha / r (lora_alpha / sqrt(r)
with rsLoRA).  This is the configuration of `train_scripts/train_pixart_lora_hf.py`: peft's `LoraConfig(r=rank,
init_lora_weights="gaussian", target_modules=[...])` with lora_alpha left at peft's default of 8, no dropout, no bias.

The adapters attach to the native modules through `convert.py`'s diffusers name mapping.  A fused native projection carries
one adapter per diffusers projection: `attn.qkv` (to_q, to_k, to_v) keeps A as [3r, K] and only the three diagonal
[C, r] blocks of B, as a [3, C, r] parameter; `cross_attn.kv_linear` (to_k, to_v) likewise with 2.  The adapter file keeps
peft's per-projection tensors.

    load_adapter(model, dir)   read `adapter_config.json` + `adapter_model.safetensors` (what `save_pretrained` writes)
    save_adapter(model, dir)   write the same files, so that `PeftModel.from_pretrained` accepts the directory
    merge_lora(model)          W <- round(W + s B A) computed in fp32; every sampler and GraphedForward then runs unchanged
    unmerge_lora(model)        restore the replaced weights bit for bit

DoRA (peft's `use_dora=True`, the reference script's `--use_dora`): `inject_dora` / `load_dora_adapter` add a trained fp32
magnitude m [N] (`lora_magnitude`, concatenated over fused projections) to every adapter.  With wn[n] = ||W[n,:] + s (B A)[n,:]||_2
taken without gradient (DoRA paper, section 4.3) and c = m / wn, a DoRA projection computes
    y = base(x) + (c - 1) * x W^T + c * s (x A^T) B^T        (peft's form; = c * (x W^T + s (x A^T) B^T) + b)
On the kernels the column-scaled GEMM applies c in its epilogue; c comes from `pxa_dora_norm` at the start of each training
forward (`prepare_operands`).  merge_lora writes W <- round(c * (W + s B A)).  This restates peft's DoRA layer; peft is not
installed here, so the restatement is not pinned against peft itself.

Training: a forward of a CUDA model with an unmerged adapter, with autograd recording, applies the adapter on the kernels
(`pixart_sigma_b200.autograd`): the down-projection u = x A^T runs as a skinny GEMM and the up-projection s u B^T as a K-tail
of the projection's own GEMM (`pxa_gemm_lora_bf16`), so that every epilogue sees the sum.  `prepare_operands` builds the bf16
operands those GEMMs read from the fp32 parameters at the start of each training forward.  The projections that run in fp32
torch (patch embedding, timestep / size embedders, t_block, final layer) apply their adapters in fp32 torch
(`linear_fp32`, `conv_fp32`).  Any other forward of a model with an unmerged adapter (no_grad, CPU, a captured
GraphedForward) raises instead of silently ignoring it.
"""
from __future__ import annotations

import json
import math
import os
from typing import Dict, Iterable, List, Optional, Tuple

import torch
from torch import nn

from . import convert

# train_pixart_lora_hf.py's target list
TARGET_MODULES = ("to_q", "to_k", "to_v", "to_out.0", "proj_in", "proj_out", "ff.net.0.proj", "ff.net.2", "proj", "linear",
                  "linear_1", "linear_2")
LORA_ALPHA = 8                     # peft's default; the reference script does not set it
CONFIG_NAME = "adapter_config.json"
WEIGHTS_NAME = "adapter_model.safetensors"
_PREFIX = "base_model.model."

_BLOCK_TARGETS = [  # (diffusers module suffix, native module suffix, group, groups)
    ("attn1.to_q", "attn.qkv", 0, 3), ("attn1.to_k", "attn.qkv", 1, 3), ("attn1.to_v", "attn.qkv", 2, 3),
    ("attn1.to_out.0", "attn.proj", 0, 1),
    ("attn2.to_q", "cross_attn.q_linear", 0, 1),
    ("attn2.to_k", "cross_attn.kv_linear", 0, 2), ("attn2.to_v", "cross_attn.kv_linear", 1, 2),
    ("attn2.to_out.0", "cross_attn.proj", 0, 1),
    ("ff.net.0.proj", "mlp.fc1", 0, 1), ("ff.net.2", "mlp.fc2", 0, 1),
]


def adaptable_modules(model: nn.Module) -> List[Tuple[str, str, int, int]]:
    """Every projection of `model` that a LoRA target can name: (diffusers module name, native module name, group, groups).
    The projections outside the blocks come first, in the order and with the names of convert.py's key mapping, then the
    blocks one by one."""
    out = []
    pairs = convert._GLOBAL + (convert._MICRO if getattr(model, "micro_conditioning", False) else [])
    for d, r in pairs:
        if d.endswith(".weight"):
            out.append((d[:-len(".weight")], r[:-len(".weight")], 0, 1))
    for i in range(len(model.blocks)):
        for d, r, g, n in _BLOCK_TARGETS:
            out.append((f"transformer_blocks.{i}.{d}", f"blocks.{i}.{r}", g, n))
    return out


def _matches(name: str, targets: Iterable[str]) -> bool:
    """peft's suffix rule for a list of target names: the module name equals a target or ends with '.' + target."""
    return any(name == t or name.endswith("." + t) for t in targets)


def _scale(r: int, alpha: float, use_rslora: bool) -> float:
    return alpha / math.sqrt(r) if use_rslora else alpha / r


def _check_config(r: int, lora_dropout: float, bias: str, use_dora: bool) -> None:
    if use_dora:
        raise NotImplementedError("DoRA adapters are created by inject_dora and read by load_dora_adapter")
    if lora_dropout:
        raise NotImplementedError("LoRA dropout is not supported (the reference script uses 0)")
    if bias != "none":
        raise NotImplementedError(f"LoRA bias={bias!r} is not supported (only 'none')")
    if r < 1:
        raise ValueError(f"LoRA rank must be positive (got {r})")


def _plan(model: nn.Module, targets: List[str]) -> Dict[str, List[str]]:
    """native module name -> the diffusers names of its adapters (one per fused projection), for every projection a target
    matches.  A fused module must be matched whole."""
    chosen: Dict[str, list] = {}
    for dname, nname, g, n in adaptable_modules(model):
        if _matches(dname, targets):
            chosen.setdefault(nname, [None] * n)[g] = dname
    for nname, groups in chosen.items():
        if any(d is None for d in groups):
            raise NotImplementedError(f"{nname}: the targets adapt only some of the projections fused in this module "
                                      f"({[d for d in groups if d]}); adapt all or none")
    return chosen


def _peft_shapes(model: nn.Module, plan: Dict[str, List[str]], r: int, dora: bool = False) -> Dict[str, Tuple[int, ...]]:
    """peft's key -> shape for every adapter tensor of `plan` (with DoRA: the magnitude too, [N] / conv [1, out, 1, 1])."""
    mods = dict(model.named_modules())
    out = {}
    for nname, groups in plan.items():
        w = mods[nname].weight
        n_g = w.shape[0] // len(groups)
        for dname in groups:
            out[f"{_PREFIX}{dname}.lora_A.weight"] = (r,) + tuple(w.shape[1:])
            out[f"{_PREFIX}{dname}.lora_B.weight"] = (n_g, r) + ((1, 1) if w.dim() == 4 else ())
            if dora:
                out[f"{_PREFIX}{dname}.lora_magnitude_vector"] = (1, n_g, 1, 1) if w.dim() == 4 else (n_g,)
    return out


def inject_lora(model: nn.Module, r: int, use_rslora: bool = False, target_modules: Iterable[str] = TARGET_MODULES,
                generator: Optional[torch.Generator] = None, *, lora_dropout: float = 0.0, bias: str = "none",
                use_dora: bool = False, lora_alpha: float = LORA_ALPHA) -> List[str]:
    """Freeze every base parameter of `model` and attach a fresh adapter to each projection a target matches.  Every check
    runs before the model is touched: a rejected call leaves it unchanged.  DoRA (use_dora=True) is `inject_dora`.

    peft's gaussian init: A ~ N(0, (1/r)^2), B = 0.  A is drawn on the CPU from `generator`, one projection after the other
    in the order of `adaptable_modules` (the projections outside the blocks, then block by block); peft draws in module
    registration order, so the distribution matches peft's but the draws for a given seed do not.  A and B are fp32
    parameters named `lora_A` / `lora_B` on the native module.  Returns the diffusers names of the adapted projections."""
    _check_config(r, lora_dropout, bias, use_dora)
    return _inject(model, r, use_rslora, list(target_modules), generator, lora_alpha)


def _inject(model, r, use_rslora, targets, generator, lora_alpha, norms=None) -> List[str]:
    if getattr(model, "_lora", None) is not None:
        raise RuntimeError("the model already carries a LoRA adapter (one adapter per model)")
    plan = _plan(model, targets)
    if norms is not None:
        norms = norms(plan)                  # DoRA: the magnitude init, checked before the model is touched
    for p in model.parameters():
        p.requires_grad_(False)
    mods = dict(model.named_modules())
    names = []
    for nname, groups in plan.items():
        mod = mods[nname]
        w = mod.weight
        G = len(groups)
        a_shape = (r,) + tuple(w.shape[1:])
        A = torch.cat([torch.randn(a_shape, generator=generator) / r for _ in range(G)], 0)
        mod.lora_A = nn.Parameter(A.to(w.device))
        mod.lora_B = nn.Parameter(torch.zeros(G, w.shape[0] // G, r, device=w.device))
        if norms is not None:
            mod.lora_magnitude = nn.Parameter(norms[nname])
        mod.__dict__["_lora_names"] = list(groups)
        mod.__dict__["_lora_scale"] = _scale(r, lora_alpha, use_rslora)
        names += groups
    model.__dict__["_lora"] = {"r": r, "alpha": lora_alpha, "use_rslora": use_rslora, "scale": _scale(r, lora_alpha, use_rslora),
                               "targets": targets, "merged": False, "dora": norms is not None}
    return names


def _row_norm_fp32(w: torch.Tensor, delta: Optional[torch.Tensor] = None) -> torch.Tensor:
    """||W[n] + delta[n]||_2 per output row in fp32 (over (in, kh, kw) for the conv), without gradient."""
    w = w.detach().float()
    if delta is not None:
        w = w + delta
    return torch.linalg.vector_norm(w.flatten(1), dim=1)


def _base_norms(model: nn.Module, plan: Dict[str, List[str]]) -> Dict[str, torch.Tensor]:
    """The DoRA magnitude init m = ||W||_row of every planned projection, on the weight's device.  On a CUDA model the
    projections that run on the GEMM kernels take it from pxa_dora_norm over the bf16 weight those GEMMs multiply (with B = 0
    the norm of each training step then reproduces it bit for bit: c = 1 exactly); the fp32 torch glue takes the fp32 norm it
    recomputes each forward.  A zero row raises: peft would compute 0 / 0 there."""
    mods = dict(model.named_modules())
    kernel = {id(m) for m in _kernel_candidates(model)}
    out = {}
    with torch.no_grad():
        for nname in plan:
            mod = mods[nname]
            w = mod.weight
            if w.is_cuda and id(mod) in kernel:
                from . import lib
                N, K = w.shape
                w16 = w.detach().to(torch.bfloat16).contiguous()
                z = lambda *shape: torch.zeros(shape, dtype=torch.bfloat16, device=w.device)
                wn = torch.empty(N, dtype=torch.float32, device=w.device)
                lib.dora_norm([(w16, z(8, K), z(N, 8), None, wn, None)], N=N, K=K, T=8)
            else:
                wn = _row_norm_fp32(w)
            if not bool((wn > 0).all()):
                raise ValueError(f"{nname}: a weight row has zero norm; DoRA's magnitude / norm is undefined there")
            out[nname] = wn
    return out


def inject_dora(model: nn.Module, r: int, use_rslora: bool = False, target_modules: Iterable[str] = TARGET_MODULES,
                generator: Optional[torch.Generator] = None, *, lora_alpha: float = LORA_ALPHA) -> List[str]:
    """`inject_lora` with DoRA (peft's `use_dora=True`): the same targets, A / B init and draw order, plus an fp32 magnitude
    `lora_magnitude` [N] per adapted projection initialised to ||W||_row, so that a fresh adapter computes the base output.
    Raises ValueError naming the module if an adapted weight row has zero norm; a rejected call leaves the model unchanged."""
    _check_config(r, 0.0, "none", False)
    return _inject(model, r, use_rslora, list(target_modules), generator, lora_alpha, norms=lambda plan: _base_norms(model, plan))


def _adapted(model: nn.Module):
    for name, mod in model.named_modules():
        if "_lora_names" in mod.__dict__:
            yield name, mod


def _state(model: nn.Module) -> dict:
    st = getattr(model, "_lora", None)
    if st is None:
        raise RuntimeError("the model carries no LoRA adapter (inject_lora / load_adapter first)")
    return st


def require_merged(model: nn.Module) -> None:
    """Raise when `model` carries an adapter whose weights are not merged: the native forward would ignore it."""
    st = model.__dict__.get("_lora")
    if st is not None and not st["merged"]:
        raise RuntimeError("PixArtMS: a LoRA adapter is attached but not merged, and the native forward does not apply "
                           "unmerged adapters; call pixart_sigma_b200.merge_lora(model) first")


def adapter_state_dict(model: nn.Module) -> Dict[str, torch.Tensor]:
    """peft's tensors for the adapter: `base_model.model.<diffusers module>.lora_{A,B}.weight`, fp32, contiguous, on the CPU.
    Linear: A [r, K], B [N, r]; the conv pos_embed.proj: A [r, 4, 2, 2], B [1152, r, 1, 1].  DoRA adds
    `<diffusers module>.lora_magnitude_vector`: [N] for a Linear, [1, 1152, 1, 1] for the conv."""
    st = _state(model)
    r = st["r"]
    out = {}
    for _, mod in _adapted(model):
        conv = mod.weight.dim() == 4
        ng = mod.lora_B.shape[1]
        for g, dname in enumerate(mod._lora_names):
            a = mod.lora_A.detach()[g * r:(g + 1) * r]
            b = mod.lora_B.detach()[g]
            if conv:
                b = b[:, :, None, None]
            out[f"{_PREFIX}{dname}.lora_A.weight"] = a.float().cpu().contiguous()
            out[f"{_PREFIX}{dname}.lora_B.weight"] = b.float().cpu().contiguous()
            if st.get("dora"):
                mg = mod.lora_magnitude.detach()[g * ng:(g + 1) * ng]
                out[f"{_PREFIX}{dname}.lora_magnitude_vector"] = (mg.view(1, ng, 1, 1) if conv else mg).float().cpu().contiguous()
    return out


def adapter_config(model: nn.Module) -> dict:
    """The `adapter_config.json` peft's `save_pretrained` writes for the reference script's LoraConfig."""
    st = _state(model)
    return {
        "alpha_pattern": {}, "auto_mapping": None, "base_model_name_or_path": None, "bias": "none", "fan_in_fan_out": False,
        "inference_mode": True, "init_lora_weights": "gaussian", "layer_replication": None, "layers_pattern": None,
        "layers_to_transform": None, "loftq_config": {}, "lora_alpha": st["alpha"], "lora_dropout": 0.0,
        "megatron_config": None, "megatron_core": "megatron.core", "modules_to_save": None, "peft_type": "LORA",
        "r": st["r"], "rank_pattern": {}, "revision": None, "target_modules": sorted(st["targets"]), "task_type": None,
        "use_dora": bool(st.get("dora")), "use_rslora": st["use_rslora"],
    }


def save_adapter(model: nn.Module, directory: str) -> None:
    """Write the adapter in peft's directory format (adapter_config.json + adapter_model.safetensors)."""
    from safetensors.torch import save_file
    os.makedirs(directory, exist_ok=True)
    sd = adapter_state_dict(model)
    with open(os.path.join(directory, CONFIG_NAME), "w") as f:
        json.dump(adapter_config(model), f, indent=2, sort_keys=True)
    save_file(sd, os.path.join(directory, WEIGHTS_NAME), metadata={"format": "pt"})


def _validate_config(cfg: dict, dora: bool = False) -> None:
    if cfg.get("peft_type") != "LORA":
        raise ValueError(f"not a LoRA adapter: peft_type={cfg.get('peft_type')!r}")
    for key in ("rank_pattern", "alpha_pattern"):
        if cfg.get(key):
            raise NotImplementedError(f"per-module {key} is not supported")
    if cfg.get("layers_to_transform") is not None or cfg.get("fan_in_fan_out"):
        raise NotImplementedError("layers_to_transform / fan_in_fan_out are not supported")
    if cfg.get("modules_to_save"):
        raise NotImplementedError("modules_to_save is not supported")
    if not isinstance(cfg.get("target_modules"), list) or not cfg["target_modules"]:
        raise ValueError("adapter_config.json: target_modules must be a non-empty list of module names")
    if dora and cfg.get("use_dora") is not True:
        raise ValueError("not a DoRA adapter (use_dora is not true): load it with load_adapter")
    _check_config(int(cfg.get("r", 0)), float(cfg.get("lora_dropout", 0.0)), cfg.get("bias", "none"),
                  bool(cfg.get("use_dora", False)) and not dora)


def load_adapter(model: nn.Module, directory: str) -> List[str]:
    """Attach the adapter stored in `directory` (peft's format) to `model`.  The config is validated, and every tensor its
    `target_modules` call for must be present with peft's shape -- no more, no fewer -- before the model is touched: a
    rejected file leaves the model unchanged.  The adapter stays unmerged; call merge_lora(model) to sample with it.
    A DoRA file (use_dora) raises NotImplementedError: it is read by load_dora_adapter."""
    return _load(model, directory, dora=False)


def load_dora_adapter(model: nn.Module, directory: str) -> List[str]:
    """`load_adapter` for a DoRA adapter (`"use_dora": true`): the same checks, plus peft's magnitude tensors
    `<diffusers module>.lora_magnitude_vector` ([N] per Linear, [1, out, 1, 1] for the conv), all before the model is touched.
    To sample with it: merge_lora(model) (e.g. `load_dora_adapter(pipe.transformer, dir); merge_lora(pipe.transformer)`)."""
    return _load(model, directory, dora=True)


def _load(model: nn.Module, directory: str, dora: bool) -> List[str]:
    from safetensors.torch import load_file
    with open(os.path.join(directory, CONFIG_NAME)) as f:
        cfg = json.load(f)
    _validate_config(cfg, dora=dora)
    if getattr(model, "_lora", None) is not None:
        raise RuntimeError("the model already carries a LoRA adapter (one adapter per model)")
    r = int(cfg["r"])
    sd = load_file(os.path.join(directory, WEIGHTS_NAME))
    want = _peft_shapes(model, _plan(model, list(cfg["target_modules"])), r, dora=dora)
    if set(sd) != set(want):
        missing, extra = sorted(set(want) - set(sd)), sorted(set(sd) - set(want))
        raise ValueError(f"adapter tensors do not match the targets: missing {missing[:4]}, unexpected {extra[:4]}")
    for k, shape in want.items():
        if tuple(sd[k].shape) != shape or not sd[k].is_floating_point():
            raise ValueError(f"{k}: {sd[k].dtype} {tuple(sd[k].shape)}, expected a floating-point tensor of shape {shape}")
    kw = dict(use_rslora=bool(cfg.get("use_rslora", False)), target_modules=cfg["target_modules"],
              lora_alpha=float(cfg.get("lora_alpha", LORA_ALPHA)))
    names = inject_dora(model, r, **kw) if dora else inject_lora(model, r, **kw)
    with torch.no_grad():
        for _, mod in _adapted(model):
            ng = mod.lora_B.shape[1]
            for g, dname in enumerate(mod._lora_names):
                mod.lora_A[g * r:(g + 1) * r].copy_(sd[f"{_PREFIX}{dname}.lora_A.weight"])
                mod.lora_B[g].copy_(sd[f"{_PREFIX}{dname}.lora_B.weight"].reshape(mod.lora_B.shape[1:]))
                if dora:
                    mod.lora_magnitude[g * ng:(g + 1) * ng].copy_(sd[f"{_PREFIX}{dname}.lora_magnitude_vector"].reshape(ng))
    return names


def _delta(mod: nn.Module, r: int, s: float) -> torch.Tensor:
    """s B A in fp32, shaped like mod.weight (block-diagonal over the fused projections)."""
    A = mod.lora_A.detach().float().flatten(1)                       # [G r, K]
    B = mod.lora_B.detach().float()                                  # [G, N/G, r]
    d = torch.cat([B[g] @ A[g * r:(g + 1) * r] for g in range(B.shape[0])], 0)
    return (s * d).view(mod.weight.shape)


def _dora_c(mod: nn.Module, delta: torch.Tensor) -> torch.Tensor:
    """c = m / ||W + s B A||_row in fp32 (no gradient), shaped to broadcast over mod.weight's rows."""
    wn = _row_norm_fp32(mod.weight, delta)
    c = mod.lora_magnitude.detach().float() / wn
    return c.view((-1,) + (1,) * (mod.weight.dim() - 1))


def merge_lora(model: nn.Module) -> None:
    """W <- W + s B A for every adapted projection (DoRA: W <- c * (W + s B A), c = m / ||W + s B A||_row): computed in fp32
    and rounded once to the parameter's dtype.  The replaced weights are kept (on the host) for unmerge_lora."""
    st = _state(model)
    if st["merged"]:
        raise RuntimeError("the LoRA adapter is already merged")
    with torch.no_grad():
        for _, mod in _adapted(model):
            w = mod.weight
            d = _delta(mod, st["r"], st["scale"])
            new = w.float() + d
            if st.get("dora"):
                new = _dora_c(mod, d) * new
            mod.__dict__["_lora_saved"] = w.detach().to("cpu", copy=True)
            w.copy_(new.to(w.dtype))
    st["merged"] = True


def unmerge_lora(model: nn.Module) -> None:
    """Restore the weights merge_lora replaced, bit for bit."""
    st = _state(model)
    if not st["merged"]:
        raise RuntimeError("the LoRA adapter is not merged")
    with torch.no_grad():
        for _, mod in _adapted(model):
            mod.weight.copy_(mod.__dict__.pop("_lora_saved"))
    st["merged"] = False


def active(mod: nn.Module) -> bool:
    """True when `mod` carries an adapter that is not merged into its weight."""
    return "_lora_names" in mod.__dict__ and "_lora_saved" not in mod.__dict__


class Operands:
    """bf16 operands of one adapted projection for the kernels, T = G r rounded up to a multiple of 8 (zero columns):
    a = A [T, K] (u = x A^T), b = s blockdiag(B) [N, T] (forward tail), at = A^T [K, T] (dgrad tail),
    bt = (s blockdiag(B))^T [T, N] (v = dY s B).  Each is rounded once from fp32.  DoRA: c = m / ||W + b a||_row (fp32 [N],
    pxa_dora_norm over the bf16 weight and these operands), else None."""
    __slots__ = ("a", "b", "at", "bt", "T", "r", "G", "s", "c")

    def __init__(self, a, b, at, bt, r, G, s, c=None):
        self.a, self.b, self.at, self.bt = a, b, at, bt
        self.T, self.r, self.G, self.s, self.c = a.shape[0], r, G, s, c


def _kernel_candidates(model: nn.Module) -> List[nn.Module]:
    """The projections that run on the GEMM kernels: every block projection and the caption projection."""
    mods = [model.y_embedder.y_proj.fc1, model.y_embedder.y_proj.fc2]
    for blk in model.blocks:
        mods += [blk.attn.qkv, blk.attn.proj, blk.cross_attn.q_linear, blk.cross_attn.kv_linear, blk.cross_attn.proj,
                 blk.mlp.fc1, blk.mlp.fc2]
    return mods


def _kernel_modules(model: nn.Module) -> List[nn.Module]:
    """The adapted projections that run on the GEMM kernels, with an unmerged adapter."""
    return [m for m in _kernel_candidates(model) if active(m)]


@torch.no_grad()
def prepare_operands(model: nn.Module) -> None:
    """(Re)build the bf16 `Operands` of every unmerged adapter on the kernel path from lora_A / lora_B, in place in buffers
    that persist across calls (so a captured training step sees optimizer updates), with a few batched ops per group of
    same-shaped projections.  Run at the start of every training forward: optimizers that write `.data` do not bump
    `_version`, so a cache keyed on it would go stale.  Projections without an active adapter lose their operands.
    DoRA: one pxa_dora_norm launch per group then writes c = m / ||W + s B A||_row for this forward (and its backward)."""
    st = model.__dict__.get("_lora")
    mods = _kernel_modules(model) if st is not None else []
    keep = set(map(id, mods))
    for m in model.modules():
        if id(m) not in keep:
            m.__dict__.pop("_pxa_lora", None)
    if not mods:
        return
    r, s, dora = st["r"], st["scale"], bool(st.get("dora"))
    if dora:
        from .autograd import _shadow
    cache = model.__dict__.setdefault("_lora_bufs", {})
    groups: Dict[tuple, List[nn.Module]] = {}
    for m in mods:
        groups.setdefault((tuple(m.lora_A.shape), tuple(m.lora_B.shape), m.weight.device), []).append(m)
    for key, ms in groups.items():
        (GR, K), (G, Ng, _), dev = key
        N, T, n = G * Ng, (GR + 7) // 8 * 8, len(ms)
        bkey = key + (n, tuple(map(id, ms)))
        bufs = cache.get(bkey)
        if bufs is None:
            z = lambda *shape: torch.zeros(shape, dtype=torch.bfloat16, device=dev)
            c = torch.ones((n, N), dtype=torch.float32, device=dev) if dora else None
            bufs = cache[bkey] = (z(n, T, K), z(n, N, T), z(n, K, T), z(n, T, N), c)
        a16, b16, at16, bt16, c32 = bufs
        A = torch.stack([m.lora_A.detach() for m in ms]).float()                  # [n, G r, K]
        sB = torch.stack([m.lora_B.detach() for m in ms]).float() * s             # [n, G, N/G, r]
        a16[:, :GR].copy_(A)
        at16[:, :, :GR].copy_(A.transpose(1, 2))
        b4, bt4 = b16.view(n, G, Ng, T), bt16.view(n, T, G, Ng)
        for g in range(G):
            b4[:, g, :, g * r:(g + 1) * r].copy_(sB[:, g])
            bt4[:, g * r:(g + 1) * r, g].copy_(sB[:, g].transpose(1, 2))
        if dora:
            mags = [m.lora_magnitude.detach() for m in ms]
            mags = [v if v.dtype == torch.float32 else v.float() for v in mags]
            from . import lib
            lib.dora_norm([(_shadow(m, "w"), a16[i], b16[i], mags[i], None, c32[i]) for i, m in enumerate(ms)], N=N, K=K, T=T)
        for i, m in enumerate(ms):
            m.__dict__["_pxa_lora"] = Operands(a16[i], b16[i], at16[i], bt16[i], r, G, s, c32[i] if dora else None)


def _dora_out(mod: nn.Module, out: torch.Tensor, base: torch.Tensor, lora: torch.Tensor, cshape) -> torch.Tensor:
    """peft's DoRA output: out + (c - 1) * base + c * lora, with base = x W^T (no bias), lora = s (x A^T) B^T and
    c = m / ||W + s B A||_row (no gradient through the norm).  c = 1 and lora = 0 leave `out` unchanged bit for bit."""
    with torch.no_grad():
        wn = _row_norm_fp32(mod.weight, _delta(mod, mod.lora_B.shape[2], mod._lora_scale))
    c = (mod.lora_magnitude.float() / wn).view(cshape)
    return out + ((c - 1) * base + c * lora)


def linear_fp32(mod: nn.Module, x: torch.Tensor) -> torch.Tensor:
    """F.linear in fp32 on `mod`'s weight, plus its unmerged adapter: x W^T + b + s (x A^T) B^T (DoRA: `_dora_out`)."""
    F = torch.nn.functional
    out = F.linear(x, mod.weight.float(), None if mod.bias is None else mod.bias.float())
    if active(mod):
        lora = mod._lora_scale * F.linear(F.linear(x, mod.lora_A.float()), mod.lora_B[0].float())
        if "lora_magnitude" not in mod._parameters:
            return out + lora
        base = F.linear(x, mod.weight.float()) if mod.bias is not None else out
        return _dora_out(mod, out, base, lora, (-1,))
    return out


def conv_fp32(mod: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
    """The patch-embedding convolution in fp32 plus its unmerged adapter: peft's lora_A is a Conv2d(in, r, k, stride) and
    lora_B a 1x1 Conv2d(r, out).  DoRA: `_dora_out` over output channels."""
    F = torch.nn.functional
    out = F.conv2d(x, mod.weight.float(), mod.bias.float(), stride=mod.stride)
    if active(mod):
        u = F.conv2d(x, mod.lora_A.float(), stride=mod.stride)
        lora = mod._lora_scale * F.conv2d(u, mod.lora_B[0].float()[:, :, None, None])
        if "lora_magnitude" not in mod._parameters:
            return out + lora
        return _dora_out(mod, out, F.conv2d(x, mod.weight.float(), stride=mod.stride), lora, (1, -1, 1, 1))
    return out
