"""Training path: the block's ops as `torch.autograd.Function`s whose forward AND backward are sm_90a kernels.

The reference trains through torch autograd (`train_scripts/train.py:197 accelerator.backward(loss)`) with per-block
activation checkpointing (`diffusion/model/utils.py:28-45`, call site `PixArtMS.py:206`).  Here autograd is only the
tape: every node below calls into libpixart_sm100.so in both directions --

  LinearFn        y = x W^T + b           bwd: dX = dY W (pxa_gemm_bf16 on the cached W^T) and dW += dY^T X (the GEMM's
                                          weight-gradient form: both activations consumed MN-major in their natural
                                          layouts, split-K, fp32 TMA reduce-add epilogue), db by pxa_colsum_bf16
  LnModulateFn    LN(x)(1+scale)+shift    bwd: pxa_ln_modulate_bwd (dx, d shift, d scale)            PixArtMS.py:75,77
  LinearGateResidualFn  x + gate*(aW^T+b) one GEMM launch (fp32 residual epilogue, aux = branch); bwd: pxa_gate_residual_bwd
                                          (d branch, d gate) then the Linear backward            PixArtMS.py:75-77
  GeluFn          gelu_tanh(pre)          bwd: pxa_gelu_tanh_bf16 with dh                            timm Mlp.act
  SelfAttnFn / CrossAttnFn / AttnKVFn     bwd: pxa_flash_attn_d72_bwd_bf16 (flash-attention-2 recomputation from lse)
                                                                                                PixArt_blocks.py:52-53,153
  KvCompressFn    LN(conv2x2s2(k | v))    bwd: pxa_kv_compress_conv2_ln_bwd                       PixArt_blocks.py:97-121

LoRA: a projection with an unmerged adapter (lora.py; operands from `lora.prepare_operands`) adds s u B^T with u = x A^T:
u is a skinny GEMM (N = T), and the up-projection is a K-tail of the projection's own GEMM (`lib.gemm(tail_a=u,
tail_w=s B)`), so every epilogue sees the sum.  Backward: v = s dY B (skinny GEMM), dX = dY W + v A (dgrad GEMM with the
tail v, A^T), dA = v^T X and dB = s dY^T u (weight-gradient form, M = T), straight into lora_A.grad / lora_B.grad when they
are bucket views.  Weights that do not require grad get no weight-gradient GEMM and no bias column sum.

Parameters may be fp32 (mixed-precision training, `train.py:369` accelerator mixed_precision) or bf16; the kernels
always consume bf16 shadows, cached per parameter version, and gradients are produced in fp32 and cast to the
parameter dtype.  There is no eager fallback: a missing library or a non-sm_100 device raises from `lib`.
"""
from __future__ import annotations

from typing import Optional

import torch

import os

from . import lib

# MLP branch as two GEMM launches with the GELU forward / backward inside their epilogues (MlpGateResidualFn), covered by
# tests/test_training_gpu.py and test_backward_gpu.py.  PXA_FUSED_MLP=0 restores the separate GELU passes.
_FUSED_MLP = os.environ.get("PXA_FUSED_MLP", "1") == "1"
# weight / bias gradients are accumulated by the kernels directly into an existing fp32 .grad (PXA_DIRECT_GRAD=0: via autograd)
_DIRECT_GRAD = os.environ.get("PXA_DIRECT_GRAD", "1") == "1"

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


def _lora_params(mod):
    """(lora_A, lora_B) of a projection with an active adapter, else (None, None): extra autograd inputs of its node."""
    return (mod.lora_A, mod.lora_B) if _lora_ops(mod) is not None else (None, None)


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
    def forward(ctx, x, weight, bias, mod, lora_A=None, lora_B=None):
        assert x.dtype == torch.bfloat16 and x.dim() == 2
        x = x.contiguous()
        out = torch.empty((x.shape[0], weight.shape[0]), dtype=torch.bfloat16, device=x.device)
        u = _lora_u(x, mod)
        lib.gemm(x, _shadow(mod, "w"), _shadow(mod, "b"), out, **_tail(u, mod, "b"))
        ctx.save_for_backward(x, weight, bias, u)
        ctx.mod = mod
        return out

    @staticmethod
    def backward(ctx, dy):
        x, weight, bias, u = ctx.saved_tensors
        n = ctx.needs_input_grad
        dx, dw, db, dA, dB = _linear_backward(n[:3], x, weight, bias, ctx.mod, dy.contiguous(), u=u, lora_needs=n[4:6])
        return dx, dw, db, None, dA, dB


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
    if p is None or not _DIRECT_GRAD:
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


class LinearGateResidualFn(torch.autograd.Function):
    """out = x32 + tab[:, i_gate] * (a W^T + b) in ONE GEMM launch (fp32 residual epilogue, PixArtMS.py:75-77): the
    branch output never makes a separate pass; with a gate it is kept (bf16 aux output of the epilogue) because the
    gate's gradient is sum_rows dout * branch."""

    @staticmethod
    def forward(ctx, a, weight, bias, mod, x32, tab, i_gate, rows_per_batch, lora_A=None, lora_B=None):
        a, x32 = a.contiguous(), x32.contiguous()
        M, N = a.shape[0], weight.shape[0]
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
        gated = i_gate >= 0
        y = torch.empty((M, N), dtype=torch.bfloat16, device=a.device) if gated else None
        u = _lora_u(a, mod)
        lib.gemm(a, _shadow(mod, "w"), _shadow(mod, "b"), out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=x32,
                 gate=tab[:, i_gate] if gated else None, gate_batch_stride=tab.stride(0) if gated else 0,
                 rows_per_batch=rows_per_batch, out_aux=y, aux_is_branch=True, **_tail(u, mod, "b"))
        ctx.save_for_backward(a, weight, bias, y, tab if gated else None, u)
        ctx.mod, ctx.idx = mod, (i_gate, rows_per_batch)
        return out

    @staticmethod
    def backward(ctx, dout):
        a, weight, bias, y, tab, u = ctx.saved_tensors
        i_gate, rpb = ctx.idx
        dout = dout.contiguous()
        dy = torch.empty(dout.shape, dtype=torch.bfloat16, device=dout.device)
        dtab = None
        if tab is not None:
            want = ctx.needs_input_grad[5]
            dg = torch.zeros((tab.shape[0], tab.shape[2]), dtype=torch.float32, device=dout.device) if want else None
            lib.gate_residual_bwd(dout, y if want else None, tab[:, i_gate], dy, dg, gate_batch_stride=tab.stride(0),
                                  rows_per_batch=rpb)
            if want:
                dtab = torch.zeros_like(tab)
                dtab[:, i_gate] = dg
        else:
            lib.gate_residual_bwd(dout, None, None, dy, None, rows_per_batch=rpb)
        n = ctx.needs_input_grad
        da, dw, db, dA, dB = _linear_backward(n[:3], a, weight, bias, ctx.mod, dy, u=u, lora_needs=n[8:10])
        return da, dw, db, None, dout, dtab, None, None, dA, dB


class MlpGateResidualFn(torch.autograd.Function):
    """The whole MLP branch
    out = x32 + gate * fc2(gelu(fc1(xn))) in TWO GEMM launches -- fc1 with the GELU epilogue that also keeps the
    pre-activation (EPI_BIAS_GELU_AUX), fc2 with the gated residual epilogue -- and a backward whose fc2 dgrad GEMM applies
    gelu'(pre) in its epilogue (EPI_MUL_DGELU): no separate GELU forward / backward passes over the [M, 4C] hidden."""

    @staticmethod
    def forward(ctx, xn, w1, b1, w2, b2, fc1, fc2, x32, tab, i_gate, rows_per_batch, A1=None, B1=None, A2=None, B2=None):
        xn, x32 = xn.contiguous(), x32.contiguous()
        M, Hd, N = xn.shape[0], w1.shape[0], w2.shape[0]
        bf = dict(dtype=torch.bfloat16, device=xn.device)
        h, pre = torch.empty((M, Hd), **bf), torch.empty((M, Hd), **bf)
        u1 = _lora_u(xn, fc1)
        lib.gemm(xn, _shadow(fc1, "w"), _shadow(fc1, "b"), h, epilogue=lib.EPI_BIAS_GELU_AUX, out_aux=pre,
                 **_tail(u1, fc1, "b"))
        out = torch.empty((M, N), dtype=torch.float32, device=xn.device)
        y = torch.empty((M, N), **bf)
        u2 = _lora_u(h, fc2)
        lib.gemm(h, _shadow(fc2, "w"), _shadow(fc2, "b"), out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=x32, gate=tab[:, i_gate],
                 gate_batch_stride=tab.stride(0), rows_per_batch=rows_per_batch, out_aux=y, aux_is_branch=True,
                 **_tail(u2, fc2, "b"))
        ctx.save_for_backward(xn, pre, h, y, tab, w1, b1, w2, b2, u1, u2)
        ctx.mods, ctx.idx = (fc1, fc2), (i_gate, rows_per_batch)
        return out

    @staticmethod
    def backward(ctx, dout):
        xn, pre, h, y, tab, w1, b1, w2, b2, u1, u2 = ctx.saved_tensors
        n = ctx.needs_input_grad
        fc1, fc2 = ctx.mods
        i_gate, rpb = ctx.idx
        dout = dout.contiguous()
        dev = dout.device
        dy = torch.empty(dout.shape, dtype=torch.bfloat16, device=dev)
        want = ctx.needs_input_grad[8]
        dg = torch.zeros((tab.shape[0], tab.shape[2]), dtype=torch.float32, device=dev) if want else None
        lib.gate_residual_bwd(dout, y if want else None, tab[:, i_gate], dy, dg, gate_batch_stride=tab.stride(0), rows_per_batch=rpb)
        dtab = None
        if want:
            dtab = torch.zeros_like(tab)
            dtab[:, i_gate] = dg
        v2 = _lora_v(dy, fc2, u2)
        _, dw2, db2, dA2, dB2 = _linear_backward((False, n[3], n[4]), h, w2, b2, fc2, dy, u=u2, v=v2, lora_needs=n[13:15])
        dpre = torch.empty_like(pre)
        lib.gemm(dy, _shadow(fc2, "t"), None, dpre, epilogue=lib.EPI_MUL_DGELU, residual=pre,     # dh * gelu'(pre) in the epilogue
                 **_tail(v2, fc2, "at"))
        dxn, dw1, db1, dA1, dB1 = _linear_backward((True, n[1], n[2]), xn, w1, b1, fc1, dpre, u=u1, lora_needs=n[11:13])
        return dxn, dw1, db1, dw2, db2, None, None, dout, dtab, None, None, dA1, dB1, dA2, dB2


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


class SelfAttnFn(torch.autograd.Function):
    """o (B*N, C) = attention over the q/k/v slices of the qkv GEMM output (B*N, 3C) (PixArt_blocks.py:130-153)."""

    @staticmethod
    def forward(ctx, qkv, B, H, N, scale, keep, fp32_p=False):
        qkv = qkv.contiguous()
        M, C3 = qkv.shape
        C = C3 // 3
        D = C // H
        q3 = qkv.view(M, 3, H, D)
        hit = keep.pop("self", None) if keep is not None and keep.get("replay") else None
        if hit is not None:                           # recomputation of a checkpointed block: (o, lse) were kept
            o, lse = hit
        else:
            o = torch.empty((M, C), dtype=torch.bfloat16, device=qkv.device)
            lse = torch.empty((B, H, N), dtype=torch.float32, device=qkv.device)
            st = (3 * C, D)
            lib.flash_attn(q3[:, 0], q3[:, 1], q3[:, 2], o, B=B, H=H, Nq=N, Nk=N, kv_rows=M, q_strides=st, k_strides=st,
                           v_strides=st, scale=scale, lse=lse, fp32_p=fp32_p)
            if keep is not None and not keep.get("replay"):
                keep["self"] = (o, lse)
        ctx.save_for_backward(qkv, o, lse)
        ctx.geom = (B, H, N, scale)
        return o

    @staticmethod
    def backward(ctx, d_o):
        qkv, o, lse = ctx.saved_tensors
        B, H, N, scale = ctx.geom
        M, C3 = qkv.shape
        C = C3 // 3
        D = C // H
        q3 = qkv.view(M, 3, H, D)
        dqkv = torch.empty_like(qkv)
        d3 = dqkv.view(M, 3, H, D)
        st = (3 * C, D)
        lib.flash_attn_bwd(q3[:, 0], q3[:, 1], q3[:, 2], o, d_o.contiguous(), lse, d3[:, 0], d3[:, 1], d3[:, 2], B=B, H=H,
                           Nq=N, Nk=N, kv_rows=M, q_strides=st, k_strides=st, v_strides=st, dq_strides=st, dk_strides=st,
                           dv_strides=st, scale=scale)
        return dqkv, None, None, None, None, None, None


class QkNormFn(torch.autograd.Function):
    """qkv (M, 3C) bf16 with q_norm / k_norm (nn.LayerNorm(C), affine) applied to the q and k slices (PixArt_blocks.py:133-134).
    Backward: the LayerNorm-modulate backward kernel with one "sample" spanning all rows, scale = weight - 1, shift = bias --
    its dscale / dshift column sums are the gradients of weight / bias."""

    @staticmethod
    def forward(ctx, qkv, qw, qb, kw, kb, eps):
        out = qkv.clone()
        C = qkv.shape[1] // 3
        bf = torch.bfloat16
        lib.layernorm_affine_(out[:, :C], qw.to(bf), qb.to(bf), eps=eps)
        lib.layernorm_affine_(out[:, C:2 * C], kw.to(bf), kb.to(bf), eps=eps)
        ctx.save_for_backward(qkv, qw, kw)
        ctx.eps = eps
        return out

    @staticmethod
    def backward(ctx, d_out):
        qkv, qw, kw = ctx.saved_tensors
        M, C3 = qkv.shape
        C = C3 // 3
        dqkv = d_out.clone()
        grads = []
        for i, w in enumerate((qw, kw)):
            x32 = qkv[:, i * C:(i + 1) * C].float().contiguous()
            dx = torch.empty_like(x32)
            dsh = torch.zeros((1, C), dtype=torch.float32, device=qkv.device)
            dsc = torch.zeros((1, C), dtype=torch.float32, device=qkv.device)
            lib.ln_modulate_bwd(x32, d_out[:, i * C:(i + 1) * C].contiguous(), (w.float() - 1.0).view(1, C).contiguous(), dx, dsh, dsc,
                                mod_batch_stride=C, rows_per_batch=M, eps=ctx.eps)
            dqkv[:, i * C:(i + 1) * C] = dx
            grads += [dsc.view(C).to(w.dtype), dsh.view(C).to(w.dtype)]
        return dqkv, grads[0], grads[1], grads[2], grads[3], None


def _qk_norm(a, qkv: torch.Tensor) -> torch.Tensor:
    if isinstance(a.q_norm, torch.nn.Identity):
        return qkv
    return QkNormFn.apply(qkv, a.q_norm.weight, a.q_norm.bias, a.k_norm.weight, a.k_norm.bias, a.q_norm.eps)


class KvCompressFn(torch.autograd.Function):
    """(kc, vc) = LN(conv2x2s2(k)), LN(conv2x2s2(v)) on the k / v slices of the qkv GEMM output (PixArt_blocks.py:97-121,
    'conv' sampling, scale factor 2).  sr = the depthwise Conv2d, norm = the LayerNorm (owners of the bf16 shadows)."""

    @staticmethod
    def forward(ctx, qkv, sr_w, sr_b, ln_w, ln_b, sr, norm, B, Hh, Ww):
        qkv = qkv.contiguous()
        M, C3 = qkv.shape
        C = C3 // 3
        n_out = (Hh // 2) * (Ww // 2)
        kc = torch.empty((B * n_out, C), dtype=torch.bfloat16, device=qkv.device)
        vc = torch.empty_like(kc)
        lib.kv_compress(qkv[:, C:2 * C], qkv[:, 2 * C:], kc.view(B, n_out, C), vc.view(B, n_out, C), _shadow(sr, "w"), _shadow(sr, "b"),
                        _shadow(norm, "w"), _shadow(norm, "b"), B=B, H=Hh, W=Ww, ld_in=C3, eps=norm.eps)
        ctx.save_for_backward(qkv, sr_w, sr_b, ln_w, ln_b)
        ctx.mods, ctx.geom = (sr, norm), (B, Hh, Ww)
        return kc, vc

    @staticmethod
    def backward(ctx, dkc, dvc):
        qkv, sr_w, sr_b, ln_w, ln_b = ctx.saved_tensors
        sr, norm = ctx.mods
        B, Hh, Ww = ctx.geom
        M, C3 = qkv.shape
        C = C3 // 3
        dqkv = torch.zeros_like(qkv)                    # the q slice gets its gradient from the attention node
        f32 = dict(dtype=torch.float32, device=qkv.device)
        g_w, g_b = torch.zeros(sr_w.shape, **f32), torch.zeros(sr_b.shape, **f32)
        g_lw, g_lb = torch.zeros(ln_w.shape, **f32), torch.zeros(ln_b.shape, **f32)
        lib.kv_compress_bwd(qkv[:, C:2 * C], qkv[:, 2 * C:], dkc.contiguous(), dvc.contiguous(), dqkv[:, C:2 * C], dqkv[:, 2 * C:],
                            _shadow(sr, "w"), _shadow(sr, "b"), _shadow(norm, "w"), g_w, g_b, g_lw, g_lb, B=B, H=Hh, W=Ww,
                            ld_in=C3, ld_din=C3, eps=norm.eps)
        return (dqkv, g_w.to(sr_w.dtype), g_b.to(sr_b.dtype), g_lw.to(ln_w.dtype), g_lb.to(ln_b.dtype), None, None, None, None, None)


class AttnKVFn(torch.autograd.Function):
    """o = attention of the q slice of qkv (B*N, 3C) over separate, already compressed keys / values (B*Nk, C)
    (KV-compressed self-attention, PixArt_blocks.py:137-153)."""

    @staticmethod
    def forward(ctx, qkv, kc, vc, B, H, N, Nk, scale, fp32_p=False):
        qkv, kc, vc = qkv.contiguous(), kc.contiguous(), vc.contiguous()
        M, C3 = qkv.shape
        C = C3 // 3
        D = C // H
        o = torch.empty((M, C), dtype=torch.bfloat16, device=qkv.device)
        lse = torch.empty((B, H, N), dtype=torch.float32, device=qkv.device)
        lib.flash_attn(qkv[:, :C], kc, vc, o, B=B, H=H, Nq=N, Nk=Nk, kv_rows=B * Nk, q_strides=(C3, D), k_strides=(C, D),
                       v_strides=(C, D), scale=scale, lse=lse, fp32_p=fp32_p)
        ctx.save_for_backward(qkv, kc, vc, o, lse)
        ctx.geom = (B, H, N, Nk, scale)
        return o

    @staticmethod
    def backward(ctx, d_o):
        qkv, kc, vc, o, lse = ctx.saved_tensors
        B, H, N, Nk, scale = ctx.geom
        M, C3 = qkv.shape
        C = C3 // 3
        D = C // H
        dqkv = torch.zeros_like(qkv)                    # k / v slices: gradient arrives through the compression node
        dkc, dvc = torch.empty_like(kc), torch.empty_like(vc)
        lib.flash_attn_bwd(qkv[:, :C], kc, vc, o, d_o.contiguous(), lse, dqkv[:, :C], dkc, dvc, B=B, H=H, Nq=N, Nk=Nk,
                           kv_rows=B * Nk, q_strides=(C3, D), k_strides=(C, D), v_strides=(C, D), dq_strides=(C3, D),
                           dk_strides=(C, D), dv_strides=(C, D), scale=scale)
        return dqkv, dkc, dvc, None, None, None, None, None, None


class CrossAttnFn(torch.autograd.Function):
    """o (B*N, C) = var-len attention of q (B*N, C) over the caption keys kv (rows, 2C) (PixArt_blocks.py:43-58)."""

    @staticmethod
    def forward(ctx, q, kv, kv_len, kv_off, B, H, N, max_keys, scale, keep):
        q, kv = q.contiguous(), kv.contiguous()
        M, C = q.shape
        D = C // H
        kv4 = kv.view(-1, 2, H, D)
        hit = keep.pop("cross", None) if keep is not None and keep.get("replay") else None
        if hit is not None:
            o, lse = hit
        else:
            o = torch.empty((M, C), dtype=torch.bfloat16, device=q.device)
            lse = torch.empty((B, H, N), dtype=torch.float32, device=q.device)
            lib.flash_attn(q, kv4[:, 0], kv4[:, 1], o, B=B, H=H, Nq=N, Nk=max_keys, kv_rows=kv.shape[0], kv_len=kv_len,
                           kv_off=kv_off, q_strides=(C, D), k_strides=(2 * C, D), v_strides=(2 * C, D), scale=scale, lse=lse)
            if keep is not None and not keep.get("replay"):
                keep["cross"] = (o, lse)
        ctx.save_for_backward(q, kv, o, lse, kv_len, kv_off)
        ctx.geom = (B, H, N, max_keys, scale)
        return o

    @staticmethod
    def backward(ctx, d_o):
        q, kv, o, lse, kv_len, kv_off = ctx.saved_tensors
        B, H, N, max_keys, scale = ctx.geom
        M, C = q.shape
        D = C // H
        kv4 = kv.view(-1, 2, H, D)
        dq = torch.empty_like(q)
        dkv = torch.zeros_like(kv)                    # rows of keys >= kv_len[b] (padding) get no gradient
        d4 = dkv.view(-1, 2, H, D)
        lib.flash_attn_bwd(q, kv4[:, 0], kv4[:, 1], o, d_o.contiguous(), lse, dq, d4[:, 0], d4[:, 1], B=B, H=H, Nq=N,
                           Nk=max_keys, kv_rows=kv.shape[0], kv_len=kv_len, kv_off=kv_off, q_strides=(C, D),
                           k_strides=(2 * C, D), v_strides=(2 * C, D), dq_strides=(C, D), dk_strides=(2 * C, D),
                           dv_strides=(2 * C, D), scale=scale)
        return dq, dkv, None, None, None, None, None, None, None, None


def linear(x: torch.Tensor, mod: torch.nn.Linear) -> torch.Tensor:
    return LinearFn.apply(x, mod.weight, mod.bias, mod, *_lora_params(mod))


def _compressed_self_attention(a, qkv: torch.Tensor, B: int, H: int, N: int, HW) -> torch.Tensor:
    """Self-attention over compressed keys / values (PixArt_blocks.py:97-121): 'conv' (scale factor 2) runs the fused
    conv + LN kernel and its backward; the parameter-free samplings are strided picks (pure data movement, torch)."""
    C = qkv.shape[1] // 3
    Hh, Ww = HW
    sr = a.sr_ratio
    if a.sampling == "conv":
        if sr != 2:
            raise NotImplementedError("conv KV compression kernel is specialised for scale_factor 2")
        kc, vc = KvCompressFn.apply(qkv, a.sr.weight, a.sr.bias, a.norm.weight, a.norm.bias, a.sr, a.norm, B, Hh, Ww)
    elif a.sampling == "uniform_every":
        kc, vc = (qkv[:, i * C:(i + 1) * C].reshape(B, N, C)[:, ::sr].reshape(-1, C) for i in (1, 2))
    elif a.sampling in ("uniform", "ave"):
        kc, vc = (qkv[:, i * C:(i + 1) * C].reshape(B, Hh, Ww, C)[:, ::sr, ::sr].reshape(-1, C) for i in (1, 2))
    else:
        raise ValueError(a.sampling)
    return AttnKVFn.apply(qkv, kc, vc, B, H, N, kc.shape[0] // B, a.scale, _fp32_p(a))


def block_forward_train(blk, x32: torch.Tensor, cond: torch.Tensor, kv_len: Optional[torch.Tensor],
                        kv_off: Optional[torch.Tensor], max_keys: int, mod: torch.Tensor, B: int, N: int,
                        keep: Optional[dict] = None, HW=None) -> torch.Tensor:
    """One PixArtMSBlock (PixArtMS.py:71-79) on the differentiable kernel ops; same arguments as `run_kernels`, but
    out of place (returns the new fp32 residual stream) so autograd / activation checkpointing can replay it.
    `keep`: per-call dict used with activation checkpointing -- the first pass stores the two attention outputs and
    their softmax statistics in it (76 MB per block at 4 x 4096 tokens), the recomputation pass (keep["replay"] set)
    takes them back instead of re-running the attention kernels."""
    a, ca, mlp = blk.attn, blk.cross_attn, blk.mlp
    H = a.num_heads
    if HW is None:
        HW = (int(N ** 0.5),) * 2
    mod = mod.contiguous()
    # (1) x += gate_msa * proj(attn(LN(x) * (1 + scale_msa) + shift_msa))                         PixArtMS.py:75
    xn = LnModulateFn.apply(x32, mod, 0, 1, N)
    if a.sr_ratio > 1:                                                       # KV token compression, PixArt_blocks.py:137-139
        ao = _compressed_self_attention(a, _qk_norm(a, linear(xn, a.qkv)), B, H, N, HW)
    else:
        ao = SelfAttnFn.apply(_qk_norm(a, linear(xn, a.qkv)), B, H, N, a.scale, keep, _fp32_p(a))
    x32 = LinearGateResidualFn.apply(ao, a.proj.weight, a.proj.bias, a.proj, x32, mod, 2, N, *_lora_params(a.proj))
    # (2) x += proj(cross_attn(x, cond))                                                          PixArtMS.py:76
    qx = linear(x32.to(torch.bfloat16), ca.q_linear)
    kv = linear(cond, ca.kv_linear)
    ao = CrossAttnFn.apply(qx, kv, kv_len, kv_off, B, H, N, max_keys, ca.head_dim ** -0.5, keep)
    x32 = LinearGateResidualFn.apply(ao, ca.proj.weight, ca.proj.bias, ca.proj, x32, mod, -1, N, *_lora_params(ca.proj))
    # (3) x += gate_mlp * fc2(gelu_tanh(fc1(LN(x) * (1 + scale_mlp) + shift_mlp)))               PixArtMS.py:77
    xn = LnModulateFn.apply(x32, mod, 3, 4, N)
    if _FUSED_MLP:                                    # experimental, see MlpGateResidualFn
        x32 = MlpGateResidualFn.apply(xn, mlp.fc1.weight, mlp.fc1.bias, mlp.fc2.weight, mlp.fc2.bias, mlp.fc1, mlp.fc2, x32, mod, 5, N,
                                      *_lora_params(mlp.fc1), *_lora_params(mlp.fc2))
    else:
        h = GeluFn.apply(linear(xn, mlp.fc1))
        x32 = LinearGateResidualFn.apply(h, mlp.fc2.weight, mlp.fc2.bias, mlp.fc2, x32, mod, 5, N, *_lora_params(mlp.fc2))
    if keep is not None:
        keep["replay"] = True            # the next call with this dict is the recomputation
    return x32


# ------------------------------------------------------------------------------------------------- the whole block as ONE node
_BLOCK_FN = os.environ.get("PXA_BLOCK_FN", "1") == "1"


_TAGS = ("qkv", "proj", "q", "kv", "cproj", "fc1", "fc2")


def _block_params(blk):
    """The block's projections in _TAGS order and, per projection, (weight, bias, lora_A, lora_B) (None: no adapter)."""
    a, ca, mlp = blk.attn, blk.cross_attn, blk.mlp
    mods = (a.qkv, a.proj, ca.q_linear, ca.kv_linear, ca.proj, mlp.fc1, mlp.fc2)
    return mods, tuple(t for m in mods for t in (m.weight, m.bias, *_lora_params(m)))


def _block_forward_kernels(blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N, kept=None):
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
        return lib.gemm(x, _shadow(lin, "w"), _shadow(lin, "b"), out, **kw, **_tail(t.get("u_" + tag), lin, "b"))

    t["xn1"] = lib.ln_modulate(x32, mod[:, 0], mod[:, 1], torch.empty((M, C), **bf), mod_batch_stride=ms, rows_per_batch=N)
    t["qkv"] = gemm("qkv", t["xn1"], a.qkv, torch.empty((M, 3 * C), **bf))
    q3 = t["qkv"].view(M, 3, H, D)
    st = (3 * C, D)
    if kept is None:
        t["ao1"], t["lse1"] = torch.empty((M, C), **bf), torch.empty((B, H, N), **f32)
        lib.flash_attn(q3[:, 0], q3[:, 1], q3[:, 2], t["ao1"], B=B, H=H, Nq=N, Nk=N, kv_rows=M, q_strides=st, k_strides=st,
                       v_strides=st, scale=a.scale, lse=t["lse1"], fp32_p=_fp32_p(a))
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
    gemm("cproj", t["ao2"], ca.proj, t["x2"], epilogue=lib.EPI_BIAS_RESIDUAL, residual=t["x1"], rows_per_batch=N)
    t["xn2"] = lib.ln_modulate(t["x2"], mod[:, 3], mod[:, 4], torch.empty((M, C), **bf), mod_batch_stride=ms, rows_per_batch=N)
    Hd = mlp.fc1.out_features
    t["h"], t["pre"] = torch.empty((M, Hd), **bf), torch.empty((M, Hd), **bf)
    gemm("fc1", t["xn2"], mlp.fc1, t["h"], epilogue=lib.EPI_BIAS_GELU_AUX, out_aux=t["pre"])
    t["x3"], t["y3"] = torch.empty((M, C), **f32), torch.empty((M, C), **bf)
    gemm("fc2", t["h"], mlp.fc2, t["x3"], epilogue=lib.EPI_BIAS_RESIDUAL, residual=t["x2"], gate=mod[:, 5], gate_batch_stride=ms,
         rows_per_batch=N, out_aux=t["y3"], aux_is_branch=True)
    return t


_SAVED = ("xn1", "qkv", "ao1", "lse1", "y1", "x1", "xb", "qx", "kv", "ao2", "lse2", "x2", "xn2", "h", "pre", "y3")
_KEPT = ("ao1", "lse1", "ao2", "lse2")


class BlockFn(torch.autograd.Function):
    """One PixArtMSBlock (PixArtMS.py:71-79, no KV compression / qk_norm) as a SINGLE autograd node: the forward is the
    kernel sequence of `_block_forward_kernels`, the backward the explicit reverse sequence of backward kernels.

    With one autograd node per op (the functions above) the training step carries ~100 small torch kernels per
    block -- zero fills and slice assignments for the modulation gradients, the gradient additions where the residual
    stream forks, bf16 casts, the accumulation of every weight gradient.
    Here the residual-stream gradient is threaded through the backward kernels (`ln_modulate_bwd(add_in=...)`,
    `gate_residual_fwd` as the fp32 + bf16 add), the six modulation gradients land in slices of ONE (6, B, C) buffer, and
    the weight / bias gradients go straight into their bucket views.  Activation checkpointing is built in (`ckpt`): only
    the block input, the conditioning and the two attention outputs + statistics are kept, the rest is recomputed here."""

    @staticmethod
    def forward(ctx, blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N, ckpt, *params):
        x32, cond, mod = x32.contiguous(), cond.contiguous(), mod.contiguous()
        t = _block_forward_kernels(blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N)
        names = (_KEPT if ckpt else _SAVED) + tuple(k for k in t if k.startswith("u_"))
        ctx.save_for_backward(x32, cond, mod, kv_len, kv_off, *[t[k] for k in names], *params)
        ctx.meta = (blk, max_keys, B, N, bool(ckpt), names)
        return t["x3"]

    @staticmethod
    def backward(ctx, dout):
        blk, max_keys, B, N, ckpt, names = ctx.meta
        saved = ctx.saved_tensors
        x32, cond, mod, kv_len, kv_off = saved[:5]
        t = dict(zip(names, saved[5:5 + len(names)]))
        params = saved[5 + len(names):]
        if ckpt:
            t = _block_forward_kernels(blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N, kept=t)
        a, ca, mlp = blk.attn, blk.cross_attn, blk.mlp
        C, H = blk.hidden_size, a.num_heads
        D, M, dev = C // H, B * N, x32.device
        bf = dict(dtype=torch.bfloat16, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        ms = mod.stride(0)
        dout = dout.contiguous()
        dm = torch.zeros((6, B, C), **f32)                # d(shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp)
        needs = ctx.needs_input_grad[10:]
        grads = {}

        def lin_bwd(tag, x, lin_mod, dy, need_dx=True, v=None):
            i = _TAGS.index(tag)
            weight, bias = params[4 * i], params[4 * i + 1]
            n = needs[4 * i:4 * i + 4]
            dx, *g = _linear_backward((need_dx, n[0], n[1]), x, weight, bias, lin_mod, dy, u=t.get("u_" + tag), v=v,
                                      lora_needs=n[2:])
            grads[tag] = g
            return dx

        # (3) x3 = x2 + gate_mlp * (fc2(gelu(fc1(xn2))) + b2)
        dy3 = torch.empty((M, C), **bf)
        lib.gate_residual_bwd(dout, t["y3"], mod[:, 5], dy3, dm[5], gate_batch_stride=ms, rows_per_batch=N)
        v2 = _lora_v(dy3, mlp.fc2, t.get("u_fc2"))
        lin_bwd("fc2", t["h"], mlp.fc2, dy3, need_dx=False, v=v2)
        dpre = torch.empty_like(t["pre"])
        lib.gemm(dy3, _shadow(mlp.fc2, "t"), None, dpre, epilogue=lib.EPI_MUL_DGELU, residual=t["pre"], **_tail(v2, mlp.fc2, "at"))
        dxn2 = lin_bwd("fc1", t["xn2"], mlp.fc1, dpre)
        dx2 = torch.empty((M, C), **f32)                  # = dout (the residual path) + the gradient through norm2
        lib.ln_modulate_bwd(t["x2"], dxn2, mod[:, 4], dx2, dm[3], dm[4], mod_batch_stride=ms, rows_per_batch=N, add_in=dout)
        # (2) x2 = x1 + cross_proj(cross_attn(q_linear(bf16(x1)), kv_linear(cond)))
        dy2 = torch.empty((M, C), **bf)
        lib.gate_residual_bwd(dx2, None, None, dy2, None, rows_per_batch=N)
        dao2 = lin_bwd("cproj", t["ao2"], ca.proj, dy2)
        dq, dkv = torch.empty((M, C), **bf), torch.zeros_like(t["kv"])      # padding key rows get no gradient
        kv4, d4 = t["kv"].view(-1, 2, H, D), dkv.view(-1, 2, H, D)
        lib.flash_attn_bwd(t["qx"], kv4[:, 0], kv4[:, 1], t["ao2"], dao2, t["lse2"], dq, d4[:, 0], d4[:, 1], B=B, H=H, Nq=N,
                           Nk=max_keys, kv_rows=t["kv"].shape[0], kv_len=kv_len, kv_off=kv_off, q_strides=(C, D),
                           k_strides=(2 * C, D), v_strides=(2 * C, D), dq_strides=(C, D), dk_strides=(2 * C, D),
                           dv_strides=(2 * C, D), scale=ca.head_dim ** -0.5)
        dxb = lin_bwd("q", t["xb"], ca.q_linear, dq)
        dcond = lin_bwd("kv", cond, ca.kv_linear, dkv)
        dx1 = torch.empty((M, C), **f32)
        lib.gate_residual_fwd(dx2, dxb, None, dx1, rows_per_batch=N)          # dx1 = dx2 + float(dxb)
        # (1) x1 = x + gate_msa * (proj(attn(qkv(xn1))) + b)
        dy1 = torch.empty((M, C), **bf)
        lib.gate_residual_bwd(dx1, t["y1"], mod[:, 2], dy1, dm[2], gate_batch_stride=ms, rows_per_batch=N)
        dao1 = lin_bwd("proj", t["ao1"], a.proj, dy1)
        dqkv = torch.empty_like(t["qkv"])
        q3, g3 = t["qkv"].view(M, 3, H, D), dqkv.view(M, 3, H, D)
        st = (3 * C, D)
        lib.flash_attn_bwd(q3[:, 0], q3[:, 1], q3[:, 2], t["ao1"], dao1, t["lse1"], g3[:, 0], g3[:, 1], g3[:, 2], B=B, H=H, Nq=N,
                           Nk=N, kv_rows=M, q_strides=st, k_strides=st, v_strides=st, dq_strides=st, dk_strides=st, dv_strides=st,
                           scale=a.scale)
        dxn1 = lin_bwd("qkv", t["xn1"], a.qkv, dqkv)
        dx = torch.empty((M, C), **f32)
        lib.ln_modulate_bwd(x32, dxn1, mod[:, 1], dx, dm[0], dm[1], mod_batch_stride=ms, rows_per_batch=N, add_in=dx1)
        pg = [g for tag in _TAGS for g in grads[tag]]
        return (None, dx, dcond, dm.permute(1, 0, 2), None, None, None, None, None, None, *pg)


def block_train(blk, x32, cond, kv_len, kv_off, max_keys, mod, B, N, HW, ckpt: bool):
    """Training forward of one block: the single-node form where it applies, else the per-op functions (with torch's
    activation checkpointing around them when `ckpt`)."""
    plain = blk.attn.sr_ratio == 1 and isinstance(blk.attn.q_norm, torch.nn.Identity)
    if _BLOCK_FN and plain:
        _, params = _block_params(blk)
        return BlockFn.apply(blk, x32, cond, mod, kv_len, kv_off, max_keys, B, N, ckpt, *params)
    if ckpt:
        from torch.utils.checkpoint import checkpoint
        return checkpoint(block_forward_train, blk, x32, cond, kv_len, kv_off, max_keys, mod, B, N, {}, HW, use_reentrant=False,
                          preserve_rng_state=False)
    return block_forward_train(blk, x32, cond, kv_len, kv_off, max_keys, mod, B, N, None, HW)
