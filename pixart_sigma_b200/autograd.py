"""Training path: `torch.autograd.Function`s whose forward AND backward are sm_90a kernels.

The reference trains through torch autograd (`train_scripts/train.py:197 accelerator.backward(loss)`) with per-block
activation checkpointing (`diffusion/model/utils.py:28-45`, call site `PixArtMS.py:206`).  Here autograd is only the
tape: every node below calls into libpixart_sm100.so in both directions --

  BlockFn         one whole PixArtMSBlock (PixArtMS.py:71-79) per node, every block kind: qk_norm (PixArt_blocks.py:133-134)
                  and KV compression (PixArt_blocks.py:97-121, 137-139) included.  Forward: the kernel sequence of
                  `_block_forward_kernels`; backward: the explicit reverse sequence (flash-attention-2 backward
                  pxa_flash_attn_d72_bwd_bf16, pxa_gate_residual_bwd, pxa_ln_modulate_bwd, pxa_kv_compress_conv2_ln_bwd and
                  the Linear backward below per projection).  Activation checkpointing is built in.

and three nodes for the glue around the blocks (caption projector and final layer, `model.PixArtMS._forward_train`):

  LinearFn        y = x W^T + b           bwd: dX = dY W (pxa_gemm_bf16 on the cached W^T) and dW += dY^T X (the GEMM's
                                          weight-gradient form: both activations consumed MN-major in their natural
                                          layouts, split-K, fp32 TMA reduce-add epilogue), db by pxa_colsum_bf16
  GeluFn          gelu_tanh(pre)          bwd: pxa_gelu_tanh_bf16 with dh                            timm Mlp.act
  LnModulateFn    LN(x)(1+scale)+shift    bwd: pxa_ln_modulate_bwd (dx, d shift, d scale)            PixArt_blocks.py:219

LoRA: a projection with an unmerged adapter (lora.py; operands from `lora.prepare_operands`) adds s u B^T with u = x A^T:
u is a skinny GEMM (N = T), and the up-projection is a K-tail of the projection's own GEMM (`lib.gemm(tail_a=u,
tail_w=s B)`), so every epilogue sees the sum.  Backward: v = s dY B (skinny GEMM), dX = dY W + v A (dgrad GEMM with the
tail v, A^T), dA = v^T X and dB = s dY^T u (weight-gradient form, M = T), straight into lora_A.grad / lora_B.grad when they
are bucket views.  Weights that do not require grad get no weight-gradient GEMM and no bias column sum.

DoRA: a projection whose adapter carries a magnitude m runs the column-scaled GEMM (`lib.gemm(col_scale=c)`, c = m / wn from
`lora.prepare_operands`): y = c (x W^T + s u B^T) + b.  Its backward first runs `lib.dora_bwd` on the gradient g of y (and the
saved y: the projection's output, its GELU pre-activation or its un-gated branch output): dz = c g in place of g, and
dm += sum_rows g (y - b) / m straight into lora_magnitude.grad when that is a bucket view.  The dgrad, v and dA / dB passes then
run unchanged on dz.

Parameters may be fp32 (mixed-precision training, `train.py:369` accelerator mixed_precision) or bf16; the kernels
always consume bf16 shadows, cached per parameter version, and gradients are produced in fp32 and cast to the
parameter dtype.  There is no eager fallback: a missing library or a non-sm_100 device raises from `lib`.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import lib
from .model import check_kv_conv_grid, kv_pick


def _shadow(mod: torch.nn.Module, kind: str) -> Optional[torch.Tensor]:
    """bf16 copy of `mod.weight` ('w'), its bf16 transpose ('t') or the bf16 bias ('b'), cached ON THE MODULE and
    rebuilt only when the parameter changed (in-place optimizer update / load_state_dict bump `_version`; `.to()` moves
    the storage).  Keyed by the owning module, not by tensor identity: under activation checkpointing autograd hands the
    backward detached aliases of the parameters, whose ids are recycled."""
    p = mod.bias if kind == "b" else mod.weight
    if p is None:
        return None
    cache = mod.__dict__.setdefault("_pxa_shadow", {})
    tag = (p._version, p.data_ptr(), p.dtype, p.device)
    hit = cache.get(kind)
    if hit is not None and hit[0] == tag:
        return hit[1]
    src = p.detach()
    old = hit[1] if hit is not None and hit[1].device == p.device and hit[1].data_ptr() != p.data_ptr() else None
    if kind == "t":
        w16 = (src if src.dtype == torch.bfloat16 else src.to(torch.bfloat16)).contiguous()
        val = lib.transpose(w16, old if old is not None and old.shape == (w16.shape[1], w16.shape[0]) else None)
    elif src.dtype == torch.bfloat16 and src.is_contiguous():
        val = src                                         # a bf16 parameter is its own shadow
    elif old is not None and old.shape == src.shape:
        val = old.copy_(src)                              # refresh in place: buffers stay valid for captured graphs
    else:
        val = src.to(torch.bfloat16).contiguous()
    cache[kind] = (tag, val)
    return val


def refresh_shadows(model: torch.nn.Module) -> None:
    """Recompute every existing bf16 shadow IN PLACE from its parameter (same buffers, new values).  Used as the first
    node of a captured training step (`training.GraphedTrainStep`): replays then see optimizer updates without any
    host-side version check."""
    tag = lambda p: (p._version, p.data_ptr(), p.dtype, p.device)
    for m in model.modules():
        cache = m.__dict__.get("_pxa_shadow")
        if not cache:
            continue
        for kind in ("w", "b"):
            if kind in cache:
                p = m.bias if kind == "b" else m.weight
                val = cache[kind][1]
                if val.data_ptr() != p.data_ptr():        # a real copy (fp32 parameter); bf16 parameters are their own shadow
                    val.copy_(p.detach())
                cache[kind] = (tag(p), val)
        if "t" in cache:
            p, val = m.weight, cache["t"][1]
            w16 = cache["w"][1] if "w" in cache else p.detach().to(torch.bfloat16).contiguous()
            lib.transpose(w16, val)
            cache["t"] = (tag(p), val)


def clear_shadow_cache(model: torch.nn.Module) -> None:
    for m in model.modules():
        m.__dict__.pop("_pxa_shadow", None)


def _lora_ops(mod):
    """The adapter operands of `mod` for this training forward (lora.Operands), or None."""
    return mod.__dict__.get("_pxa_lora")


def _is_dora(mod) -> bool:
    op = _lora_ops(mod)
    return op is not None and op.c is not None


def _lora_params(mod):
    """(lora_A, lora_B, lora_magnitude) of a projection with an active adapter (magnitude None without DoRA), else
    (None, None, None): extra autograd inputs of its node."""
    if _lora_ops(mod) is None:
        return (None, None, None)
    return (mod.lora_A, mod.lora_B, mod.lora_magnitude if _is_dora(mod) else None)


def _scale(mod) -> dict:
    """gemm() arguments of the DoRA column scale of `mod`, if any."""
    return dict(col_scale=_lora_ops(mod).c) if _is_dora(mod) else {}


def _dora_bwd(mod, g, y, need_m: bool, inplace: bool):
    """(dz, dm) of a DoRA projection for the gradient g of its output y = c z + b: dz = c g (over g when `inplace`) and the
    magnitude gradient, added into lora_magnitude.grad when the kernel may accumulate there (then dm is None).  Without DoRA:
    (g, None)."""
    if not _is_dora(mod):
        return g, None
    mag = mod.lora_magnitude
    m32 = mag.detach() if mag.dtype == torch.float32 else mag.detach().float()
    acc = _grad_accumulator(mag) if need_m else None
    dm = acc if acc is not None else torch.zeros(mag.shape, dtype=torch.float32, device=g.device)
    dz = g if inplace else torch.empty_like(g)
    lib.dora_bwd(g, y, _shadow(mod, "b"), _lora_ops(mod).c, m32, dz, dm)
    if acc is not None:
        _grad_landed(mag)
        return dz, None
    return dz, (dm if mag.dtype == torch.float32 else dm.to(mag.dtype)) if need_m else None


def _lora_u(x, mod):
    """u = x A^T (bf16 [M, T]) for the forward tail, or None."""
    op = _lora_ops(mod)
    if op is None:
        return None
    return lib.gemm(x, op.a, None, torch.empty((x.shape[0], op.T), dtype=torch.bfloat16, device=x.device))


def _lora_v(dy, mod, u):
    """v = s dY B (bf16 [M, T]) for the dgrad tail, or None (no adapter: u is None)."""
    if u is None:
        return None
    op = _lora_ops(mod)
    return lib.gemm(dy, op.bt, None, torch.empty((dy.shape[0], op.T), dtype=torch.bfloat16, device=dy.device))


def _tail(t, mod, kind: str) -> dict:
    """gemm() arguments of the K-tail t [M, T] times the adapter operand `kind` of `mod` ("b" forward, "at" dgrad)."""
    return {} if t is None else dict(tail_a=t, tail_w=getattr(_lora_ops(mod), kind))


def _to_grad(p, g):
    """Add the fp32 gradient g into p.grad when the kernels may accumulate there directly, else return it for autograd."""
    acc = _grad_accumulator(p)
    if acc is None:
        return g if p.dtype == torch.float32 else g.to(p.dtype)
    acc.add_(g)
    _grad_landed(p)
    return None


def _lora_wgrad(mod, x, u, dy, v, needs):
    """(dA, dB) of the adapter of `mod`: dA = v^T x and dB = s dY^T u on the diagonal blocks.  needs = (A, B)."""
    op = _lora_ops(mod)
    A, B = mod.lora_A, mod.lora_B
    dA = dB = None
    dev = x.device
    GR = A.shape[0]
    if needs[0]:
        acc = _grad_accumulator(A)
        if acc is not None and op.T == GR:
            lib.gemm_wgrad(v, x, acc)                                          # straight into the bucket view
            _grad_landed(A)
        else:
            g = torch.zeros((op.T, x.shape[1]), dtype=torch.float32, device=dev)
            lib.gemm_wgrad(v, x, g)
            dA = _to_grad(A, g[:GR])
    if needs[1]:
        G, Ng, r = B.shape
        g = torch.zeros((op.T, dy.shape[1]), dtype=torch.float32, device=dev)  # u^T dY: only its diagonal blocks are used
        lib.gemm_wgrad(u, dy, g)
        blocks = g[:GR].view(G, r, G, Ng).diagonal(dim1=0, dim2=2).permute(2, 1, 0)    # [G, Ng, r]
        dB = _to_grad(B, blocks * op.s)
    return dA, dB


class LinearFn(torch.autograd.Function):
    """y = x W^T + b of `mod` (an nn.Linear: the owner of the bf16 shadows); weight / bias (and the adapter's lora_A /
    lora_B) are passed as tensors too so that autograd routes their gradients."""

    @staticmethod
    def forward(ctx, x, weight, bias, mod, lora_A=None, lora_B=None, lora_magnitude=None):
        assert x.dtype == torch.bfloat16 and x.dim() == 2
        x = x.contiguous()
        out = torch.empty((x.shape[0], weight.shape[0]), dtype=torch.bfloat16, device=x.device)
        u = _lora_u(x, mod)
        lib.gemm(x, _shadow(mod, "w"), _shadow(mod, "b"), out, **_tail(u, mod, "b"), **_scale(mod))
        ctx.save_for_backward(x, weight, bias, u, out if _is_dora(mod) else None)
        ctx.mod = mod
        return out

    @staticmethod
    def backward(ctx, dy):
        x, weight, bias, u, y = ctx.saved_tensors
        n = ctx.needs_input_grad
        dz, dm = _dora_bwd(ctx.mod, dy.contiguous(), y, n[6], inplace=False)
        dx, dw, db, dA, dB = _linear_backward(n[:3], x, weight, bias, ctx.mod, dz, u=u, lora_needs=n[4:6])
        return dx, dw, db, None, dA, dB, dm


def _linear_backward(ctx_needs, x, weight, bias, mod, dy, u=None, v=None, lora_needs=(False, False)):
    """(dx, dw, db, dA, dB) of y = x W^T + b [+ s (x A^T) B^T] for the incoming dy (bf16, contiguous); ctx_needs =
    needs_input_grad of (x, W, b), lora_needs of (A, B).  u = x A^T from the forward (None: no adapter); v = s dY B when
    the caller already has it."""
    M, K = x.shape
    N = weight.shape[0]
    dx = dw = db = dA = dB = None
    lora = u is not None and (ctx_needs[0] or any(lora_needs))
    if lora and v is None:
        v = _lora_v(dy, mod, u)
    if ctx_needs[0]:
        dx = torch.empty((M, K), dtype=torch.bfloat16, device=x.device)
        # dX = dY . W (+ v A)   (W^T is K-contiguous in N)
        lib.gemm(dy, _shadow(mod, "t"), None, dx, **_tail(v if lora else None, mod, "at"))
    if ctx_needs[1]:
        acc = _grad_accumulator(mod.weight)
        if acc is not None:
            # the weight-gradient GEMM's TMA reduce-add epilogue accumulates STRAIGHT into the parameter's fp32 .grad (a view
            # of its gradient bucket): no zero-filled temporary, no autograd accumulation pass (~10 GB of HBM traffic / step)
            lib.gemm_wgrad(dy, x, acc)
            _grad_landed(mod.weight)
        else:
            dw32 = torch.zeros((N, K), dtype=torch.float32, device=x.device)
            lib.gemm_wgrad(dy, x, dw32)                                        # dW += dY^T . X  (MN-major operands, split-K)
            dw = dw32 if weight.dtype == torch.float32 else dw32.to(weight.dtype)
    if bias is not None and ctx_needs[2]:
        acc = _grad_accumulator(mod.bias)
        if acc is not None:
            lib.colsum(dy, acc)
            _grad_landed(mod.bias)
        else:
            db32 = torch.zeros((N,), dtype=torch.float32, device=x.device)
            lib.colsum(dy, db32)
            db = db32 if bias.dtype == torch.float32 else db32.to(bias.dtype)
    if lora and any(lora_needs):
        dA, dB = _lora_wgrad(mod, x, u, dy, v, lora_needs)
    return dx, dw, db, dA, dB


def _grad_accumulator(p: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """The tensor a backward kernel may accumulate a parameter gradient into directly: the parameter's existing fp32,
    contiguous `.grad` (e.g. its view into a `parallel.GradBucketReducer` bucket).  None -> hand the gradient to autograd."""
    if p is None:
        return None
    g = p.grad
    if g is None or g.dtype != torch.float32 or not g.is_contiguous() or g.device != p.device or g.shape != p.shape:
        return None
    return g


def _grad_landed(p: torch.Tensor) -> None:
    """Tell whoever tracks gradient readiness (GradBucketReducer) that p.grad has received this backward's contribution --
    the job autograd's post-accumulate hook does for gradients that go through autograd."""
    cb = getattr(p, "_pxa_grad_ready", None)
    if cb is not None:
        cb()


class LnModulateFn(torch.autograd.Function):
    """xn = LN(x) * (1 + mod[:, i_scale]) + mod[:, i_shift]; x (B*N, C) fp32, mod (B, G, C) fp32 contiguous."""

    @staticmethod
    def forward(ctx, x32, mod, i_shift, i_scale, rows_per_batch):
        assert x32.dtype == torch.float32 and mod.dtype == torch.float32 and mod.is_contiguous()
        x32 = x32.contiguous()
        xn = torch.empty(x32.shape, dtype=torch.bfloat16, device=x32.device)
        lib.ln_modulate(x32, mod[:, i_shift], mod[:, i_scale], xn, mod_batch_stride=mod.stride(0), rows_per_batch=rows_per_batch)
        ctx.save_for_backward(x32, mod)
        ctx.idx = (i_shift, i_scale, rows_per_batch)
        return xn

    @staticmethod
    def backward(ctx, dxn):
        x32, mod = ctx.saved_tensors
        i_shift, i_scale, rpb = ctx.idx
        B, G, C = mod.shape
        dx = torch.empty_like(x32)
        dsh = torch.zeros((B, C), dtype=torch.float32, device=x32.device)
        dsc = torch.zeros((B, C), dtype=torch.float32, device=x32.device)
        lib.ln_modulate_bwd(x32, dxn.contiguous(), mod[:, i_scale], dx, dsh, dsc, mod_batch_stride=mod.stride(0),
                            rows_per_batch=rpb)
        dmod = None
        if ctx.needs_input_grad[1]:
            dmod = torch.zeros_like(mod)
            dmod[:, i_shift] = dsh
            dmod[:, i_scale] = dsc
        return dx, dmod, None, None, None


class GeluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pre):
        pre = pre.contiguous()
        ctx.save_for_backward(pre)
        return lib.gelu_tanh(pre)

    @staticmethod
    def backward(ctx, dh):
        (pre,) = ctx.saved_tensors
        return lib.gelu_tanh(pre, dh=dh.contiguous())


def _fp32_p(attn) -> bool:
    """`fp32_attention` (set on every submodule by `set_grad_checkpoint`, model/utils.py:31-34; read by AttentionKVCompress only,
    PixArt_blocks.py:145-147): the forward P V takes P as bf16 hi + lo terms (PxaAttnArgs.p_precision = 1).  The backward
    kernel recomputes P from the same fp32 statistics and keeps its bf16 operands (gradient bars: tests/test_backward_gpu.py)."""
    return bool(getattr(attn, "fp32_attention", False))


def linear(x: torch.Tensor, mod: torch.nn.Linear) -> torch.Tensor:
    return LinearFn.apply(x, mod.weight, mod.bias, mod, *_lora_params(mod))


# ------------------------------------------------------------------------------------------------- the whole block as ONE node
_TAGS = ("qkv", "proj", "q", "kv", "cproj", "fc1", "fc2")


def _norms_qk(a) -> bool:
    return not isinstance(a.q_norm, torch.nn.Identity)


_PER = 5                                            # BlockFn inputs per projection


def _block_params(blk):
    """The block's parameters as BlockFn inputs: per projection in _TAGS order (weight, bias, lora_A, lora_B,
    lora_magnitude) (None: no adapter / no DoRA), then (weight, bias) of q_norm and k_norm (qk_norm) and of sr and norm (conv
    KV compression) where the block has them.  A plain block has 35."""
    a, ca, mlp = blk.attn, blk.cross_attn, blk.mlp
    mods = (a.qkv, a.proj, ca.q_linear, ca.kv_linear, ca.proj, mlp.fc1, mlp.fc2)
    extra = ((a.q_norm, a.k_norm) if _norms_qk(a) else ()) + ((a.sr, a.norm) if a.sr_ratio > 1 and a.sampling == "conv" else ())
    return tuple(t for m in mods for t in (m.weight, m.bias, *_lora_params(m))) + tuple(t for m in extra for t in (m.weight, m.bias))


def _compress_kv(a, qkv, B, N, HW):
    """(kc, vc) (B*Nk, C): the compressed keys / values of the qkv GEMM output.  'conv' (scale factor 2) runs the fused
    conv + LN kernel; the parameter-free samplings are strided picks (`model.kv_pick`, pure data movement, torch)."""
    C3 = qkv.shape[1]
    C = C3 // 3
    k, v = qkv[:, C:2 * C], qkv[:, 2 * C:]
    if a.sampling != "conv":
        return tuple(kv_pick(x, B, HW, a.sampling, a.sr_ratio).contiguous().view(-1, C) for x in (k, v))
    check_kv_conv_grid(HW, a.sr_ratio)
    Hh, Ww = HW
    n_out = (Hh // 2) * (Ww // 2)
    kc = torch.empty((B * n_out, C), dtype=torch.bfloat16, device=qkv.device)
    vc = torch.empty_like(kc)
    lib.kv_compress(k, v, kc.view(B, n_out, C), vc.view(B, n_out, C), _shadow(a.sr, "w"), _shadow(a.sr, "b"),
                    _shadow(a.norm, "w"), _shadow(a.norm, "b"), B=B, H=Hh, W=Ww, ld_in=C3, eps=a.norm.eps)
    return kc, vc


def _compress_kv_bwd(a, qkv, dkc, dvc, dqkv, B, N, HW):
    """Backward of `_compress_kv`: the gradients of kc / vc into the k / v slices of dqkv (zero-filled by the caller).  Returns
    the fp32 gradients of sr.weight, sr.bias, norm.weight, norm.bias ('conv'), else []."""
    C3 = qkv.shape[1]
    C = C3 // 3
    if a.sampling != "conv":
        for d, dx in ((dkc, dqkv[:, C:2 * C]), (dvc, dqkv[:, 2 * C:])):
            pick = kv_pick(dx, B, HW, a.sampling, a.sr_ratio)
            pick.copy_(d.view(pick.shape))
        return []
    g = [torch.zeros(p.shape, dtype=torch.float32, device=qkv.device) for p in (a.sr.weight, a.sr.bias, a.norm.weight, a.norm.bias)]
    lib.kv_compress_bwd(qkv[:, C:2 * C], qkv[:, 2 * C:], dkc, dvc, dqkv[:, C:2 * C], dqkv[:, 2 * C:], _shadow(a.sr, "w"),
                        _shadow(a.sr, "b"), _shadow(a.norm, "w"), *g, B=B, H=HW[0], W=HW[1], ld_in=C3, ld_din=C3, eps=a.norm.eps)
    return g


def _self_kv(t, B, H, N):
    """(k, v, their (row, head) strides, Nk) of the self-attention: the k / v slices of qkv, or the compressed kc / vc."""
    M, C3 = t["qkv"].shape
    D = C3 // 3 // H
    if "kc" in t:
        return t["kc"], t["vc"], (C3 // 3, D), t["kc"].shape[0] // B
    q3 = t["qkv"].view(M, 3, H, D)
    return q3[:, 1], q3[:, 2], (C3, D), N


def _block_forward_kernels(blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N, HW, kept=None):
    """The block's forward on the kernels, out of place, returning every intermediate the backward reads.  `kept` = the two
    attention outputs + softmax statistics of an earlier pass and its adapter down-projections u_<tag> (activation
    checkpointing: they are not recomputed)."""
    a, ca, mlp = blk.attn, blk.cross_attn, blk.mlp
    C, H = blk.hidden_size, a.num_heads
    D, M, dev = C // H, B * N, x32.device
    bf = dict(dtype=torch.bfloat16, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    ms = mod.stride(0)
    t = {k: v for k, v in kept.items() if k.startswith("u_")} if kept is not None else {}

    def gemm(tag, x, lin, out, **kw):
        """The projection `lin` (tag in _TAGS) with its adapter's up-projection as the K-tail; u_<tag> kept in t."""
        if _lora_ops(lin) is not None and "u_" + tag not in t:
            t["u_" + tag] = _lora_u(x, lin)
        return lib.gemm(x, _shadow(lin, "w"), _shadow(lin, "b"), out, **kw, **_tail(t.get("u_" + tag), lin, "b"), **_scale(lin))

    t["xn1"] = lib.ln_modulate(x32, mod[:, 0], mod[:, 1], torch.empty((M, C), **bf), mod_batch_stride=ms, rows_per_batch=N)
    t["qkv"] = gemm("qkv", t["xn1"], a.qkv, torch.empty((M, 3 * C), **bf))
    if _norms_qk(a):                                  # q_norm / k_norm, PixArt_blocks.py:133-134; the backward reads qkv_pre
        t["qkv_pre"], t["qkv"] = t["qkv"], t["qkv"].clone()
        for i, ln in enumerate((a.q_norm, a.k_norm)):
            lib.layernorm_affine_(t["qkv"][:, i * C:(i + 1) * C], _shadow(ln, "w"), _shadow(ln, "b"), eps=ln.eps)
    if a.sr_ratio > 1:                                # KV token compression, PixArt_blocks.py:137-139
        t["kc"], t["vc"] = _compress_kv(a, t["qkv"], B, N, HW)
    q3 = t["qkv"].view(M, 3, H, D)
    st = (3 * C, D)
    if kept is None:
        k, v, kst, Nk = _self_kv(t, B, H, N)
        t["ao1"], t["lse1"] = torch.empty((M, C), **bf), torch.empty((B, H, N), **f32)
        lib.flash_attn(q3[:, 0], k, v, t["ao1"], B=B, H=H, Nq=N, Nk=Nk, kv_rows=B * Nk, q_strides=st, k_strides=kst,
                       v_strides=kst, scale=a.scale, lse=t["lse1"], fp32_p=_fp32_p(a))
    else:
        t["ao1"], t["lse1"] = kept["ao1"], kept["lse1"]
    t["x1"], t["y1"] = torch.empty((M, C), **f32), torch.empty((M, C), **bf)
    gemm("proj", t["ao1"], a.proj, t["x1"], epilogue=lib.EPI_BIAS_RESIDUAL, residual=x32, gate=mod[:, 2], gate_batch_stride=ms,
         rows_per_batch=N, out_aux=t["y1"], aux_is_branch=True)
    t["xb"] = t["x1"].to(torch.bfloat16)
    t["qx"] = gemm("q", t["xb"], ca.q_linear, torch.empty((M, C), **bf))
    t["kv"] = gemm("kv", cond, ca.kv_linear, torch.empty((cond.shape[0], 2 * C), **bf))
    kv4 = t["kv"].view(-1, 2, H, D)
    if kept is None:
        t["ao2"], t["lse2"] = torch.empty((M, C), **bf), torch.empty((B, H, N), **f32)
        lib.flash_attn(t["qx"], kv4[:, 0], kv4[:, 1], t["ao2"], B=B, H=H, Nq=N, Nk=max_keys, kv_rows=cond.shape[0], kv_len=kv_len,
                       kv_off=kv_off, q_strides=(C, D), k_strides=(2 * C, D), v_strides=(2 * C, D), scale=ca.head_dim ** -0.5,
                       lse=t["lse2"])
    else:
        t["ao2"], t["lse2"] = kept["ao2"], kept["lse2"]
    t["x2"] = torch.empty((M, C), **f32)
    if _is_dora(ca.proj):                             # its DoRA backward reads the branch output c z + b
        t["y2"] = torch.empty((M, C), **bf)
    gemm("cproj", t["ao2"], ca.proj, t["x2"], epilogue=lib.EPI_BIAS_RESIDUAL, residual=t["x1"], rows_per_batch=N,
         **(dict(out_aux=t["y2"], aux_is_branch=True) if "y2" in t else {}))
    t["xn2"] = lib.ln_modulate(t["x2"], mod[:, 3], mod[:, 4], torch.empty((M, C), **bf), mod_batch_stride=ms, rows_per_batch=N)
    Hd = mlp.fc1.out_features
    t["h"], t["pre"] = torch.empty((M, Hd), **bf), torch.empty((M, Hd), **bf)
    gemm("fc1", t["xn2"], mlp.fc1, t["h"], epilogue=lib.EPI_BIAS_GELU_AUX, out_aux=t["pre"])
    t["x3"], t["y3"] = torch.empty((M, C), **f32), torch.empty((M, C), **bf)
    gemm("fc2", t["h"], mlp.fc2, t["x3"], epilogue=lib.EPI_BIAS_RESIDUAL, residual=t["x2"], gate=mod[:, 5], gate_batch_stride=ms,
         rows_per_batch=N, out_aux=t["y3"], aux_is_branch=True)
    return t


_SAVED = ("xn1", "qkv", "ao1", "lse1", "y1", "x1", "xb", "qx", "kv", "ao2", "lse2", "x2", "xn2", "h", "pre", "y3")
_SAVED_EXTRA = ("qkv_pre", "kc", "vc", "y2")        # only blocks with qk_norm / KV compression / a DoRA cross_attn.proj
_KEPT = ("ao1", "lse1", "ao2", "lse2")


class BlockFn(torch.autograd.Function):
    """One PixArtMSBlock (PixArtMS.py:71-79) as a SINGLE autograd node: the forward is the kernel sequence of
    `_block_forward_kernels`, the backward the explicit reverse sequence of backward kernels.

    One autograd node per op would carry ~100 small torch kernels per block -- zero fills and slice assignments for the
    modulation gradients, the gradient additions where the residual stream forks, bf16 casts, the accumulation of every
    weight gradient.  Here the residual-stream gradient is threaded through the backward kernels
    (`ln_modulate_bwd(add_in=...)`, `gate_residual_fwd` as the fp32 + bf16 add), the six modulation gradients land in
    slices of ONE (6, B, C) buffer, and the weight / bias gradients of the projections go straight into their bucket views
    (those of q_norm / k_norm / sr / norm go through autograd).  Activation checkpointing is built in (`ckpt`): only the
    block input, the conditioning and the two attention outputs + statistics are kept, the rest (compressed keys / values
    included) is recomputed here."""

    @staticmethod
    def forward(ctx, blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N, HW, ckpt, *params):
        x32, cond, mod = x32.contiguous(), cond.contiguous(), mod.contiguous()
        t = _block_forward_kernels(blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N, HW)
        names = (_KEPT if ckpt else _SAVED + tuple(k for k in _SAVED_EXTRA if k in t)) + tuple(k for k in t if k.startswith("u_"))
        ctx.save_for_backward(x32, cond, mod, kv_len, kv_off, *[t[k] for k in names], *params)
        ctx.meta = (blk, max_keys, B, N, HW, bool(ckpt), names)
        return t["x3"]

    @staticmethod
    def backward(ctx, dout):
        blk, max_keys, B, N, HW, ckpt, names = ctx.meta
        saved = ctx.saved_tensors
        x32, cond, mod, kv_len, kv_off = saved[:5]
        t = dict(zip(names, saved[5:5 + len(names)]))
        params = saved[5 + len(names):]
        if ckpt:
            t = _block_forward_kernels(blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N, HW, kept=t)
        a, ca, mlp = blk.attn, blk.cross_attn, blk.mlp
        C, H = blk.hidden_size, a.num_heads
        D, M, dev = C // H, B * N, x32.device
        bf = dict(dtype=torch.bfloat16, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        ms = mod.stride(0)
        dout = dout.contiguous()
        dm = torch.zeros((6, B, C), **f32)                # d(shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp)
        needs = ctx.needs_input_grad[11:]
        grads, dmag = {}, {}

        def lin_bwd(tag, x, lin_mod, dy, need_dx=True, v=None):
            i = _TAGS.index(tag)
            weight, bias = params[_PER * i], params[_PER * i + 1]
            n = needs[_PER * i:_PER * i + 4]
            dx, *g = _linear_backward((need_dx, n[0], n[1]), x, weight, bias, lin_mod, dy, u=t.get("u_" + tag), v=v,
                                      lora_needs=n[2:])
            grads[tag] = g
            return dx

        def dora(tag, lin_mod, g, y):
            """DoRA: g (the gradient of the projection's output y) becomes dz = c g in place; the magnitude gradient."""
            dmag[tag] = _dora_bwd(lin_mod, g, y, needs[_PER * _TAGS.index(tag) + 4], inplace=True)[1]

        # (3) x3 = x2 + gate_mlp * (fc2(gelu(fc1(xn2))) + b2)
        dy3 = torch.empty((M, C), **bf)
        lib.gate_residual_bwd(dout, t["y3"], mod[:, 5], dy3, dm[5], gate_batch_stride=ms, rows_per_batch=N)
        dora("fc2", mlp.fc2, dy3, t["y3"])
        v2 = _lora_v(dy3, mlp.fc2, t.get("u_fc2"))
        lin_bwd("fc2", t["h"], mlp.fc2, dy3, need_dx=False, v=v2)
        dpre = torch.empty_like(t["pre"])
        lib.gemm(dy3, _shadow(mlp.fc2, "t"), None, dpre, epilogue=lib.EPI_MUL_DGELU, residual=t["pre"], **_tail(v2, mlp.fc2, "at"))
        dora("fc1", mlp.fc1, dpre, t["pre"])
        dxn2 = lin_bwd("fc1", t["xn2"], mlp.fc1, dpre)
        dx2 = torch.empty((M, C), **f32)                  # = dout (the residual path) + the gradient through norm2
        lib.ln_modulate_bwd(t["x2"], dxn2, mod[:, 4], dx2, dm[3], dm[4], mod_batch_stride=ms, rows_per_batch=N, add_in=dout)
        # (2) x2 = x1 + cross_proj(cross_attn(q_linear(bf16(x1)), kv_linear(cond)))
        dy2 = torch.empty((M, C), **bf)
        lib.gate_residual_bwd(dx2, None, None, dy2, None, rows_per_batch=N)
        dora("cproj", ca.proj, dy2, t.get("y2"))
        dao2 = lin_bwd("cproj", t["ao2"], ca.proj, dy2)
        dq, dkv = torch.empty((M, C), **bf), torch.zeros_like(t["kv"])      # padding key rows get no gradient
        kv4, d4 = t["kv"].view(-1, 2, H, D), dkv.view(-1, 2, H, D)
        lib.flash_attn_bwd(t["qx"], kv4[:, 0], kv4[:, 1], t["ao2"], dao2, t["lse2"], dq, d4[:, 0], d4[:, 1], B=B, H=H, Nq=N,
                           Nk=max_keys, kv_rows=t["kv"].shape[0], kv_len=kv_len, kv_off=kv_off, q_strides=(C, D),
                           k_strides=(2 * C, D), v_strides=(2 * C, D), dq_strides=(C, D), dk_strides=(2 * C, D),
                           dv_strides=(2 * C, D), scale=ca.head_dim ** -0.5)
        dora("q", ca.q_linear, dq, t["qx"])
        dora("kv", ca.kv_linear, dkv, t["kv"])
        dxb = lin_bwd("q", t["xb"], ca.q_linear, dq)
        dcond = lin_bwd("kv", cond, ca.kv_linear, dkv)
        dx1 = torch.empty((M, C), **f32)
        lib.gate_residual_fwd(dx2, dxb, None, dx1, rows_per_batch=N)          # dx1 = dx2 + float(dxb)
        # (1) x1 = x + gate_msa * (proj(attn(qkv(xn1))) + b)
        dy1 = torch.empty((M, C), **bf)
        lib.gate_residual_bwd(dx1, t["y1"], mod[:, 2], dy1, dm[2], gate_batch_stride=ms, rows_per_batch=N)
        dora("proj", a.proj, dy1, t["y1"])
        dao1 = lin_bwd("proj", t["ao1"], a.proj, dy1)
        compressed = a.sr_ratio > 1
        dqkv = torch.zeros_like(t["qkv"]) if compressed else torch.empty_like(t["qkv"])  # k / v rows no kept key reads: 0
        q3, g3 = t["qkv"].view(M, 3, H, D), dqkv.view(M, 3, H, D)
        st = (3 * C, D)
        k, v, kst, Nk = _self_kv(t, B, H, N)
        dk, dv = (torch.empty_like(k), torch.empty_like(v)) if compressed else (g3[:, 1], g3[:, 2])
        lib.flash_attn_bwd(q3[:, 0], k, v, t["ao1"], dao1, t["lse1"], g3[:, 0], dk, dv, B=B, H=H, Nq=N, Nk=Nk, kv_rows=B * Nk,
                           q_strides=st, k_strides=kst, v_strides=kst, dq_strides=st, dk_strides=kst, dv_strides=kst,
                           scale=a.scale)
        kv_grads = _compress_kv_bwd(a, t["qkv"], dk, dv, dqkv, B, N, HW) if compressed else []
        qk_grads = []
        if _norms_qk(a):
            # LN-modulate backward with one "sample" spanning all rows and scale = weight - 1: its dscale / dshift column sums
            # are the gradients of weight / bias.  The weight is the bf16 shadow the forward's layernorm_affine_ used, not an
            # fp32 master weight: dx is the derivative of the function the forward computed (w - 1 is exact in fp32).
            for i, ln in enumerate((a.q_norm, a.k_norm)):
                xs = t["qkv_pre"][:, i * C:(i + 1) * C].float().contiguous()
                dxs = torch.empty_like(xs)
                dsh, dsc = torch.zeros((1, C), **f32), torch.zeros((1, C), **f32)
                scale = (_shadow(ln, "w").float() - 1.0).view(1, C)
                lib.ln_modulate_bwd(xs, dqkv[:, i * C:(i + 1) * C].contiguous(), scale, dxs, dsh, dsc, mod_batch_stride=C,
                                    rows_per_batch=M, eps=ln.eps)
                dqkv[:, i * C:(i + 1) * C] = dxs
                qk_grads += [dsc.view(C), dsh.view(C)]
        dora("qkv", a.qkv, dqkv, t["qkv_pre"] if _norms_qk(a) else t["qkv"])
        dxn1 = lin_bwd("qkv", t["xn1"], a.qkv, dqkv)
        dx = torch.empty((M, C), **f32)
        lib.ln_modulate_bwd(x32, dxn1, mod[:, 1], dx, dm[0], dm[1], mod_batch_stride=ms, rows_per_batch=N, add_in=dx1)
        pg = [g for tag in _TAGS for g in grads[tag] + [dmag[tag]]]
        np_ = _PER * len(_TAGS)
        pg += [g.to(p.dtype) if n else None for g, p, n in zip(qk_grads + kv_grads, params[np_:], needs[np_:])]
        return (None, dx, dcond, dm.permute(1, 0, 2), None, None, None, None, None, None, None, *pg)


def block_train(blk, x32, cond, kv_len, kv_off, max_keys, mod, B, N, HW, ckpt: bool):
    """Training forward of one block: one BlockFn node, activation-checkpointed when `ckpt`."""
    return BlockFn.apply(blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N, tuple(HW), ckpt, *_block_params(blk))
