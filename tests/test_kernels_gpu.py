"""GPU parity tests (-m gpu) of the individual sm_90a kernels, called through the C-ABI (ctypes), against the
oracle's fp32 restatement of the same op evaluated on the same bf16-rounded inputs.

Tolerances (normwise ||a-b||/||b||, stated per test): a bf16 result carries 2^-9 relative rounding per element
(~1.7e-3 normwise), so bf16-output kernels are held to 4e-3 and the fp32-residual path to 2e-4.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
DEV = "cuda"


def _randn(*shape, seed=0, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


# ------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K,bn", [
    (128, 192, 64, 0), (256, 384, 1152, 0), (1000, 1152, 1152, 0), (4096, 3456, 1152, 0), (300, 2304, 1152, 0),
    (512, 1152, 4608, 0), (384, 256, 128, 256), (384, 256, 128, 128), (200, 200, 200, 192), (200, 200, 200, 128),
    (130, 32, 1152, 128),
])
def test_gemm_bias_bf16(M, N, K, bn):
    a, w, bias = _randn(M, K, seed=1), _randn(N, K, seed=2, scale=K ** -0.5), _randn(N, seed=3, scale=0.1)
    out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS, block_n=bn)
    want = F.linear(a.float(), w.float(), bias.float())
    assert po.rel_err(out.float(), want) < 4e-3


@pytest.mark.parametrize("M,N,K,bn", [(256, 192, 64, 192), (512, 384, 1152, 192), (1000, 1152, 1152, 192),
                                      (4096, 3456, 1152, 192), (300, 2304, 1152, 0), (640, 4608, 1152, 256),
                                      (384, 256, 128, 128), (200, 200, 200, 192)])
@pytest.mark.parametrize("rev", [False, True])
def test_gemm_bias_bf16_tile_widths(M, N, K, bn, rev):
    a, w, bias = _randn(M, K, seed=1), _randn(N, K, seed=2, scale=K ** -0.5), _randn(N, seed=3, scale=0.1)
    out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS, block_n=bn, reverse_tiles=rev)
    want = F.linear(a.float(), w.float(), bias.float())
    assert po.rel_err(out.float(), want) < 4e-3


def test_gemm_many_tiles_gelu_and_residual():
    M, N, K = 2048, 1152, 1152
    a, w, bias = _randn(M, K, seed=4), _randn(N, K, seed=5, scale=K ** -0.5), _randn(N, seed=6, scale=0.1)
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_GELU, max_ctas=6)     # 6 CTAs walk 16 x 6 tiles
    want = F.gelu(F.linear(a.float(), w.float(), bias.float()), approximate="tanh")
    assert po.rel_err(out.float(), want) < 4e-3
    x = _randn(M, N, seed=7, dtype=torch.float32)
    gate = _randn(2, 6, N, seed=8, dtype=torch.float32)
    want = x + gate[:, 2].repeat_interleave(M // 2, 0) * F.linear(a.float(), w.float(), bias.float())
    lib.gemm(a, w, bias, x, epilogue=lib.EPI_BIAS_RESIDUAL, residual=x, gate=gate[:, 2], gate_batch_stride=6 * N,
             rows_per_batch=M // 2)
    assert po.rel_err(x, want) < 2e-4


def test_gemm_many_tiles_per_cta_and_no_bias():
    """3 CTAs walk 8x6 tiles: exercises smem-ring phase wrap-around."""
    M, N, K = 1024, 1152, 1152
    a, w = _randn(M, K, seed=4), _randn(N, K, seed=5, scale=K ** -0.5)
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    lib.gemm(a, w, None, out, max_ctas=3)
    assert po.rel_err(out.float(), a.float() @ w.float().T) < 4e-3


def test_gemm_gelu_tanh():
    M, N, K = 2048, 4608, 1152
    a, w, bias = _randn(M, K, seed=6), _randn(N, K, seed=7, scale=K ** -0.5), _randn(N, seed=8, scale=0.1)
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_GELU)
    want = F.gelu(F.linear(a.float(), w.float(), bias.float()), approximate="tanh")
    assert po.rel_err(out.float(), want) < 4e-3


@pytest.mark.parametrize("out_dtype,tol", [(torch.float32, 2e-4), (torch.bfloat16, 4e-3)])
@pytest.mark.parametrize("gated", [True, False])
def test_gemm_gate_residual(out_dtype, tol, gated):
    B, Ntok, N, K = 3, 400, 1152, 4608            # M = 1200: M tail + rows_per_batch not a tile multiple
    M = B * Ntok
    a, w, bias = _randn(M, K, seed=9), _randn(N, K, seed=10, scale=K ** -0.5), _randn(N, seed=11, scale=0.1)
    res = _randn(M, N, seed=12, dtype=out_dtype)
    mod = _randn(B, 6, N, seed=13, dtype=torch.float32)
    gate = mod[:, 2] if gated else None
    out = torch.empty(M, N, dtype=out_dtype, device=DEV)
    aux = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=res, gate=gate, gate_batch_stride=6 * N,
             rows_per_batch=Ntok, out_aux=aux)
    y = F.linear(a.float(), w.float(), bias.float())
    if gated:
        y = y * mod[:, 2].repeat_interleave(Ntok, 0)
    want = res.float() + y
    assert po.rel_err(out.float(), want) < tol
    assert po.rel_err(aux.float(), want) < 4e-3


def test_gemm_gate_residual_samples_shorter_than_a_tile():
    """96 tokens per sample (< the 128-row tile): a tile spans up to three samples, per-row gate lookup."""
    B, Ntok, N, K = 5, 96, 1152, 1152
    M = B * Ntok
    a, w, bias = _randn(M, K, seed=9), _randn(N, K, seed=10, scale=K ** -0.5), _randn(N, seed=11, scale=0.1)
    x = _randn(M, N, seed=12, dtype=torch.float32)
    mod = _randn(B, 6, N, seed=13, dtype=torch.float32)
    want = x + mod[:, 5].repeat_interleave(Ntok, 0) * F.linear(a.float(), w.float(), bias.float())
    lib.gemm(a, w, bias, x, epilogue=lib.EPI_BIAS_RESIDUAL, residual=x, gate=mod[:, 5], gate_batch_stride=6 * N,
             rows_per_batch=Ntok)
    assert po.rel_err(x, want) < 2e-4


def test_gemm_residual_in_place():
    M, N, K = 512, 1152, 1152
    a, w = _randn(M, K, seed=14), _randn(N, K, seed=15, scale=K ** -0.5)
    x = _randn(M, N, seed=16, dtype=torch.float32)
    want = x + a.float() @ w.float().T
    lib.gemm(a, w, None, x, epilogue=lib.EPI_BIAS_RESIDUAL, residual=x)
    assert po.rel_err(x, want) < 2e-4


@pytest.mark.parametrize("bn", [128, 192, 256])
@pytest.mark.parametrize("mode", ["aux", "in_place"])
@pytest.mark.parametrize("rev", [False, True])
def test_gemm_residual_chunk_ring_parity(bn, mode, rev):
    """fp32 residual epilogue: 3 CTAs walk 8 x ceil(1184/bn) tiles whose last column tile has an odd number of 32-column
    chunks, so the two epilogue warpgroups swap chunk parity from tile to tile and the 4-deep chunk ring wraps many
    times; both the load/store path (bf16 aux copy) and the TMA reduce-add path (in place, no aux)."""
    M, N, K = 1000, 1184, 1152
    a, w, bias = _randn(M, K, seed=21), _randn(N, K, seed=22, scale=K ** -0.5), _randn(N, seed=23, scale=0.1)
    x = _randn(M, N, seed=24, dtype=torch.float32)
    gate = _randn(2, 6, N, seed=25, dtype=torch.float32)
    want = x + gate[:, 4].repeat_interleave(M // 2, 0) * F.linear(a.float(), w.float(), bias.float())
    kw = dict(epilogue=lib.EPI_BIAS_RESIDUAL, residual=x, gate=gate[:, 4], gate_batch_stride=6 * N, rows_per_batch=M // 2,
              block_n=bn, max_ctas=3, reverse_tiles=rev)
    if mode == "aux":
        aux = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        lib.gemm(a, w, bias, x, out_aux=aux, **kw)
        assert po.rel_err(aux.float(), want) < 4e-3
    else:
        lib.gemm(a, w, bias, x, **kw)
    assert po.rel_err(x, want) < 2e-4


def test_gemm_rejects_bad_arguments():
    a, w = _randn(128, 64), _randn(192, 64)
    out = torch.empty(128, 192, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(lib.PxaError):
        lib.gemm(a, w, None, out, block_n=100)
    with pytest.raises(lib.PxaError):
        lib.gemm(a, w, None, out, epilogue=lib.EPI_BIAS_RESIDUAL)     # residual missing


# ------------------------------------------------------------------------------------------------- LN + modulate
@pytest.mark.parametrize("B,Ntok", [(3, 333), (5, 1001)])     # the second: more rows than resident warps (grid-stride + prefetch)
@pytest.mark.parametrize("xdtype", [torch.float32, torch.bfloat16])
def test_ln_modulate(xdtype, B, Ntok):
    Cc = 1152
    x = (_randn(B * Ntok, Cc, seed=20, dtype=torch.float32) * 3 + 0.5).to(xdtype)
    mod = _randn(B, 6, Cc, seed=21, dtype=torch.float32)
    out = torch.empty(B * Ntok, Cc, dtype=torch.bfloat16, device=DEV)
    lib.ln_modulate(x, mod[:, 3], mod[:, 4], out, mod_batch_stride=6 * Cc, rows_per_batch=Ntok)
    want = po.ln_modulate(x.float().view(B, Ntok, Cc), mod[:, 3:4], mod[:, 4:5]).view(-1, Cc)
    assert po.rel_err(out.float(), want) < 4e-3
    out2 = torch.empty_like(out)
    lib.ln_modulate(x, mod[:, 3], mod[:, 4], out2, mod_batch_stride=6 * Cc, rows_per_batch=Ntok, reverse_rows=True)
    assert torch.equal(out, out2)                                   # row order only


# ------------------------------------------------------------------------------------------------- fused LN-modulate chain
def _ln_reference(x, shift, scale, w, bias, rows_per_batch, gelu):
    """F.linear(LN(x) * (1 + scale_b) + shift_b, w, bias) in fp32 -- what norm + t2i_modulate + Linear compute
    (PixArtMS.py:75,77; PixArt_blocks.py:24-25)."""
    B = x.shape[0] // rows_per_batch
    xn = po.ln_modulate(x.view(B, rows_per_batch, -1), shift[:, None], scale[:, None]).reshape(x.shape)
    y = F.linear(xn, w.float(), bias.float())
    return F.gelu(y, approximate="tanh") if gelu else y


def _uv(w, bias, shift, scale):
    """u_b = W (1 + scale_b), v_b = W shift_b + bias in fp32 (the per-sample vectors of PXA_EPI_LN_BIAS)."""
    return (1.0 + scale) @ w.float().T, shift @ w.float().T + bias.float()


def test_ln_prepare_scaled_copy_and_row_sums():
    B, Ntok, Cc = 3, 200, 1152
    x = _randn(B * Ntok, Cc, seed=50, dtype=torch.float32) * 2 + 0.3
    mod = _randn(B, 6, Cc, seed=51, dtype=torch.float32) * 0.3
    a = torch.empty(B * Ntok, Cc, dtype=torch.bfloat16, device=DEV)
    stats = torch.full((B * Ntok, lib.LN_STAT_PARTS, 2), float("nan"), device=DEV)
    lib.ln_prepare(x, mod[:, 4], a, stats, mod_batch_stride=6 * Cc, rows_per_batch=Ntok)
    want = x * mod[:, 4].repeat_interleave(Ntok, 0)
    assert po.rel_err(a.float(), want) < 4e-3
    assert po.rel_err(stats.sum(1)[:, 0], x.sum(1)) < 1e-5 and po.rel_err(stats.sum(1)[:, 1], (x * x).sum(1)) < 1e-5
    assert torch.equal(stats[:, 1:], torch.zeros_like(stats[:, 1:]))


@pytest.mark.parametrize("N,gelu,rpb", [(3456, False, 1024), (4608, True, 1024), (3456, False, 200), (1152, True, 333),
                                       (384, False, 2048)])
def test_gemm_ln_epilogue_matches_norm_modulate_linear(N, gelu, rpb):
    """EPI_LN_BIAS(_GELU): LayerNorm + modulate folded into the GEMM epilogue vs the unfused fp32 computation.  Row groups of
    200 / 333 rows put sample boundaries inside 128-row tiles (two staged u / v rows per tile)."""
    B, K = 2, 1152
    M = B * rpb
    x = _randn(M, K, seed=52, dtype=torch.float32) * 1.7 + _randn(M, 1, seed=53, dtype=torch.float32) * 0.5
    shift = _randn(B, K, seed=54, dtype=torch.float32) * 0.3
    scale = _randn(B, K, seed=55, dtype=torch.float32) * 0.3
    w, bias = _randn(N, K, seed=56, scale=K ** -0.5), _randn(N, seed=57, scale=0.1)
    a = torch.empty(M, K, dtype=torch.bfloat16, device=DEV)
    stats = torch.empty(M, lib.LN_STAT_PARTS, 2, device=DEV)
    lib.ln_prepare(x, (1 + scale).contiguous(), a, stats, mod_batch_stride=K, rows_per_batch=rpb)
    u, v = _uv(w, bias, shift, scale)
    out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
    lib.gemm(a, w, None, out, epilogue=lib.EPI_LN_BIAS_GELU if gelu else lib.EPI_LN_BIAS, rows_per_batch=rpb,
             ln_stats=stats, ln_u=u.contiguous(), ln_v=v.contiguous(), ln_uv_batch_stride=N, ln_dim=K, ln_eps=1e-6)
    want = _ln_reference(x, shift, scale, w, bias, rpb, gelu)
    assert torch.isfinite(out.float()).all()
    assert po.rel_err(out.float(), want) < 4e-3


@pytest.mark.parametrize("K,byp", [(1152, True), (1152, False), (4608, True), (4608, False)])
@pytest.mark.parametrize("rev", [False, True])
def test_gemm_residual_epilogue_scaled_aux_and_row_stats(K, byp, rev):
    """The fp32 residual epilogue as the PRODUCER of the fused LayerNorm: x_new = x + gate (a W^T + b) (checked as before),
    out_aux = bf16(x_new * aux_scale_b), row_stats_out = per-column-tile partial (sum, sum of squares) of x_new.
    byp False: the same epilogue without the by-products, result only."""
    B, rpb, N = 3, 1000, 1152
    M = B * rpb
    a, w, bias = _randn(M, K, seed=60), _randn(N, K, seed=61, scale=K ** -0.5), _randn(N, seed=62, scale=0.1)
    x = _randn(M, N, seed=63, dtype=torch.float32)
    gate = _randn(B, 6, N, seed=64, dtype=torch.float32)
    asc = 1 + _randn(B, 2, N, seed=65, dtype=torch.float32) * 0.3
    want = x + gate[:, 2].repeat_interleave(rpb, 0) * F.linear(a.float(), w.float(), bias.float())
    aux = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV) if byp else None
    stats = torch.full((M, lib.LN_STAT_PARTS, 2), float("nan"), device=DEV) if byp else None
    lib.gemm(a, w, bias, x, epilogue=lib.EPI_BIAS_RESIDUAL, residual=x, gate=gate[:, 2], gate_batch_stride=6 * N,
             rows_per_batch=rpb, reverse_tiles=rev, out_aux=aux, aux_scale=asc[:, 1] if byp else None,
             aux_scale_batch_stride=2 * N, row_stats_out=stats)
    assert po.rel_err(x, want) < 2e-4
    if byp:
        assert po.rel_err(aux.float(), want * asc[:, 1].repeat_interleave(rpb, 0)) < 4e-3
        assert torch.isfinite(stats).all()
        assert po.rel_err(stats.sum(1)[:, 0], want.sum(1)) < 1e-3           # sums of ~N(0,1) values: absolute error ~1e-4
        assert po.rel_err(stats.sum(1)[:, 1], (want * want).sum(1)) < 1e-4


def test_fused_ln_chain_producer_to_consumer():
    """Producer epilogue -> consumer epilogue end to end: (x + a W1^T) normalised, modulated and projected by W2 without a
    stand-alone LayerNorm pass, against the fp32 computation of the same two layers."""
    B, rpb, C, N2 = 2, 1024, 1152, 4608
    M = B * rpb
    a, w1, b1 = _randn(M, C, seed=70), _randn(C, C, seed=71, scale=C ** -0.5), _randn(C, seed=72, scale=0.1)
    w2, b2 = _randn(N2, C, seed=73, scale=C ** -0.5), _randn(N2, seed=74, scale=0.1)
    x = _randn(M, C, seed=75, dtype=torch.float32) + 0.4
    shift, scale = _randn(B, C, seed=76, dtype=torch.float32) * 0.3, _randn(B, C, seed=77, dtype=torch.float32) * 0.3
    x_new = x + F.linear(a.float(), w1.float(), b1.float())
    want = _ln_reference(x_new, shift, scale, w2, b2, rpb, True)
    xs = torch.empty(M, C, dtype=torch.bfloat16, device=DEV)
    stats = torch.empty(M, lib.LN_STAT_PARTS, 2, device=DEV)
    lib.gemm(a, w1, b1, x, epilogue=lib.EPI_BIAS_RESIDUAL, residual=x, rows_per_batch=rpb, out_aux=xs,
             aux_scale=(1 + scale).contiguous(), aux_scale_batch_stride=C, row_stats_out=stats)
    u, v = _uv(w2, b2, shift, scale)
    out = torch.empty(M, N2, dtype=torch.bfloat16, device=DEV)
    lib.gemm(xs, w2, None, out, epilogue=lib.EPI_LN_BIAS_GELU, rows_per_batch=rpb, ln_stats=stats, ln_u=u.contiguous(),
             ln_v=v.contiguous(), ln_uv_batch_stride=N2, ln_dim=C)
    assert po.rel_err(x, x_new) < 2e-4
    assert po.rel_err(out.float(), want) < 5e-3


def test_layernorm_affine_inplace_on_qkv_slices():
    """qk_norm (PixArt_blocks.py:133-134): LayerNorm(C, affine, eps 1e-5) on the q and k column slices of the qkv buffer."""
    M, Cc = 777, 1152
    qkv = _randn(M, 3 * Cc, seed=80) * 2
    w, b = (1 + _randn(Cc, seed=81, scale=0.1).float()).to(torch.bfloat16), _randn(Cc, seed=82, scale=0.1)
    want_q = F.layer_norm(qkv[:, :Cc].float(), (Cc,), w.float(), b.float(), eps=1e-5)
    v_before = qkv[:, 2 * Cc:].clone()
    lib.layernorm_affine_(qkv[:, :Cc], w, b, eps=1e-5)
    assert po.rel_err(qkv[:, :Cc].float(), want_q) < 4e-3
    assert torch.equal(qkv[:, 2 * Cc:], v_before)


# ------------------------------------------------------------------------------------------------- attention
def _attn_ref(q, k, v, lens):
    """oracle sdpa per sample on fp32 copies; q (B,Nq,H,72), k/v (B,Nk,H,72); lens = valid keys per sample."""
    outs = []
    for b, L in enumerate(lens):
        if L == 0:
            outs.append(torch.zeros_like(q[b:b + 1]).float())
        else:
            outs.append(po.sdpa_heads(q[b:b + 1].float(), k[b:b + 1, :L].float(), v[b:b + 1, :L].float()))
    return torch.cat(outs, 0)


@pytest.mark.parametrize("B,H,Nq,Nk", [(1, 1, 128, 128), (1, 2, 256, 256), (2, 16, 1024, 1024), (1, 16, 1000, 1000),
                                       (2, 4, 1024, 256), (1, 3, 300, 77)])
@pytest.mark.parametrize("fp32_p", [False, True])
@pytest.mark.parametrize("rev", [False, True])
def test_flash_attn_self_from_qkv_layout(B, H, Nq, Nk, fp32_p, rev):
    """q/k/v are strided views of a (B*N, 3, H, 72)-style buffer exactly as the QKV GEMM leaves them."""
    q = _randn(B, Nq, H, 72, seed=30)
    k = _randn(B, Nk, H, 72, seed=31)
    v = _randn(B, Nk, H, 72, seed=32)
    out = torch.full((B * Nq, H * 72), float("nan"), dtype=torch.bfloat16, device=DEV)
    lib.flash_attn(q, k, v, out, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=B * Nk,
                   q_strides=(H * 72, 72), k_strides=(H * 72, 72), v_strides=(H * 72, 72),
                   fp32_p=fp32_p, reverse_batch=rev)
    want = _attn_ref(q, k, v, [Nk] * B).reshape(B * Nq, H * 72)
    assert torch.isfinite(out.float()).all()
    assert po.rel_err(out.float(), want) < 6e-3


@pytest.mark.parametrize("fp32_p", [False, True])
@pytest.mark.parametrize("rev", [False, True])
def test_flash_attn_interleaved_qkv_buffer(fp32_p, rev):
    B, H, N = 2, 16, 512
    qkv = _randn(B * N, 3, H, 72, seed=33)
    out = torch.empty(B * N, H * 72, dtype=torch.bfloat16, device=DEV)
    lib.flash_attn(qkv[:, 0], qkv[:, 1], qkv[:, 2], out, B=B, H=H, Nq=N, Nk=N, kv_rows=B * N,
                   q_strides=(3 * H * 72, 72), k_strides=(3 * H * 72, 72), v_strides=(3 * H * 72, 72),
                   fp32_p=fp32_p, reverse_batch=rev)
    r = qkv.view(B, N, 3, H, 72)
    want = _attn_ref(r[:, :, 0], r[:, :, 1], r[:, :, 2], [N] * B).reshape(B * N, H * 72)
    assert po.rel_err(out.float(), want) < 6e-3


@pytest.mark.parametrize("fp32_p", [False, True])
@pytest.mark.parametrize("rev", [False, True])
def test_flash_attn_large_logits_trigger_rescale(fp32_p, rev):
    """Keys ordered so the running max keeps growing from block to block: every block's O / l rescale by corr changes the
    result."""
    B, H, N = 1, 2, 512
    q = _randn(B, N, H, 72, seed=34)
    k = _randn(B, N, H, 72, seed=35)
    ramp = torch.linspace(0.2, 6.0, N, device=DEV).view(1, N, 1, 1)
    k = (k.float() * ramp).to(torch.bfloat16)
    v = _randn(B, N, H, 72, seed=36)
    out = torch.empty(B * N, H * 72, dtype=torch.bfloat16, device=DEV)
    lib.flash_attn(q, k, v, out, B=B, H=H, Nq=N, Nk=N, kv_rows=B * N, q_strides=(H * 72, 72), k_strides=(H * 72, 72),
                   v_strides=(H * 72, 72), fp32_p=fp32_p, reverse_batch=rev)
    want = _attn_ref(q, k, v, [N]).reshape(B * N, H * 72)
    assert po.rel_err(out.float(), want) < 8e-3


@pytest.mark.parametrize("fp32_p", [False, True])
@pytest.mark.parametrize("rev", [False, True])
def test_flash_attn_cross_packed_varlen(fp32_p, rev):
    """T5 cross-attention: packed keys (1, sum L, 2, H, 72) with BlockDiagonalMask semantics, incl. an empty sample."""
    H, Nq = 16, 384
    lens = [300, 8, 0, 129, 128, 77]
    B = len(lens)
    tot = sum(lens)
    q = _randn(B, Nq, H, 72, seed=37)
    kv = _randn(tot, 2, H, 72, seed=38)
    off = torch.tensor([sum(lens[:i]) for i in range(B)], dtype=torch.int32, device=DEV)
    ln = torch.tensor(lens, dtype=torch.int32, device=DEV)
    out = torch.full((B * Nq, H * 72), float("nan"), dtype=torch.bfloat16, device=DEV)
    lib.flash_attn(q, kv[:, 0], kv[:, 1], out, B=B, H=H, Nq=Nq, Nk=300, kv_rows=tot, kv_len=ln, kv_off=off,
                   q_strides=(H * 72, 72), k_strides=(2 * H * 72, 72), v_strides=(2 * H * 72, 72),
                   fp32_p=fp32_p, reverse_batch=rev)
    wants, o = [], 0
    for b, L in enumerate(lens):
        if L == 0:
            wants.append(torch.zeros(1, Nq, H, 72, device=DEV))
        else:
            wants.append(po.sdpa_heads(q[b:b + 1].float(), kv[None, o:o + L, 0].float(), kv[None, o:o + L, 1].float()))
        o += L
    want = torch.cat(wants, 0).reshape(B * Nq, H * 72)
    assert torch.isfinite(out.float()).all()
    assert po.rel_err(out.float(), want) < 6e-3


# ------------------------------------------------------------------------------------------------- KV compression
def test_kv_compress_conv2_ln():
    B, Hh, Ww, Cc = 2, 16, 24, 1152
    qkv = _randn(B * Hh * Ww, 3 * Cc, seed=40)
    sd = {"a.sr.weight": _randn(Cc, 1, 2, 2, seed=41, scale=0.3), "a.sr.bias": _randn(Cc, seed=42, scale=0.1),
          "a.norm.weight": (1 + _randn(Cc, seed=43, scale=0.1).float()).to(torch.bfloat16),
          "a.norm.bias": _randn(Cc, seed=44, scale=0.1)}
    ko = torch.empty(B, Hh * Ww // 4, Cc, dtype=torch.bfloat16, device=DEV)
    vo = torch.empty_like(ko)
    lib.kv_compress(qkv[:, Cc:2 * Cc], qkv[:, 2 * Cc:], ko, vo, sd["a.sr.weight"], sd["a.sr.bias"], sd["a.norm.weight"],
                    sd["a.norm.bias"], B=B, H=Hh, W=Ww, ld_in=3 * Cc)
    sdf = {k_: v_.float() for k_, v_ in sd.items()}
    for got, col in ((ko, 1), (vo, 2)):
        src = qkv[:, col * Cc:(col + 1) * Cc].float().view(B, Hh * Ww, Cc)
        want = po.kv_downsample(sdf, "a", src, Hh, Ww, 2, "conv")
        assert po.rel_err(got.float(), want) < 4e-3


# ------------------------------------------------------------------------------------------------- skinny GEMMs (M < one tile)
@pytest.mark.parametrize("M,N", [(4, 3456), (16, 8064), (64, 16128), (130, 4608)])
def test_gemm_few_rows_fp32_accumulate_in_place(M, N):
    """The per-forward conditioning GEMMs of the fused LayerNorm (model._LnFusion): a handful of rows against tall weight
    stacks, fp32 result accumulated in place through the TMA reduce-add epilogue."""
    K = 1152
    a, w = _randn(M, K, seed=90), _randn(N, K, seed=91, scale=K ** -0.5)
    out = torch.zeros(M, N, device=DEV)
    lib.gemm(a, w, None, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=out)
    want = a.float() @ w.float().T
    assert po.rel_err(out, want) < 1e-5
    lib.gemm(a, w, None, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=out)          # accumulates
    assert po.rel_err(out, 2 * want) < 1e-5


def test_ln_fusion_conditioning_vectors_match_fp32():
    """model._LnFusion.prepare: u = W (1 + scale), v = W shift + bias for (qkv | fc1) of every block, against fp32 torch."""
    from pixart_sigma_b200.model import PixArtMSBlock, _LnFusion, _Workspace
    torch.manual_seed(3)
    with torch.device(DEV):
        blocks = [PixArtMSBlock(1152, 16).to(torch.bfloat16) for _ in range(2)]
    B, Cc = 3, 1152
    t0 = _randn(B, 6, Cc, seed=92, dtype=torch.float32) * 0.3
    mod_all = torch.stack([b.scale_shift_table.float()[None] + t0 for b in blocks])
    u, v, one_plus = _LnFusion(blocks).prepare(t0, mod_all, _Workspace())
    for i, b in enumerate(blocks):
        for lin, sl, i_shift, i_scale in ((b.attn.qkv, slice(0, 3456), 0, 1), (b.mlp.fc1, slice(3456, 8064), 3, 4)):
            want_u = (1 + mod_all[i, :, i_scale]) @ lin.weight.float().T
            want_v = mod_all[i, :, i_shift] @ lin.weight.float().T + lin.bias.float()
            assert po.rel_err(u[i][:, sl], want_u) < 1e-5 and po.rel_err(v[i][:, sl], want_v) < 1e-5
    assert torch.equal(one_plus[:, :, 0], 1 + mod_all[:, :, 1]) and torch.equal(one_plus[:, :, 1], 1 + mod_all[:, :, 4])


# ------------------------------------------------------------------------------------------------- L2 chaining options
@pytest.mark.parametrize("epi", ["bias", "residual"])
def test_gemm_reverse_tile_order_gives_identical_results(epi):
    """reverse_tiles only changes the order in which the persistent grid visits the tiles (last row block first)."""
    M, N, K = 2304, 1152, 4608
    a, w, bias = _randn(M, K, seed=100), _randn(N, K, seed=101, scale=K ** -0.5), _randn(N, seed=102, scale=0.1)
    outs = []
    for rev in (False, True):
        if epi == "bias":
            out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=DEV)
            lib.gemm(a, w, bias, out, reverse_tiles=rev)
        else:
            out = _randn(M, N, seed=103, dtype=torch.float32)
            gate = _randn(2, N, seed=104, dtype=torch.float32)
            lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=out, gate=gate, gate_batch_stride=N,
                     rows_per_batch=M // 2, reverse_tiles=rev)
        outs.append(out)
    assert torch.isfinite(outs[1].float()).all()
    if epi == "bias":
        assert torch.equal(outs[0], outs[1])
    else:
        assert po.rel_err(outs[1], outs[0]) < 1e-6        # TMA reduce-add: same addends, L2 adds them in arrival order


@pytest.mark.parametrize("fp32_p", [False, True])
@pytest.mark.parametrize("with_lse", [False, True])
def test_flash_attn_reverse_batch_order_gives_identical_results(fp32_p, with_lse):
    B, H, N = 3, 4, 640
    q, k, v = _randn(B, N, H, 72, seed=110), _randn(B, N, H, 72, seed=111), _randn(B, N, H, 72, seed=112)
    lens = torch.tensor([640, 77, 300], dtype=torch.int32, device=DEV)
    outs, lses = [], []
    for rev in (False, True):
        out = torch.full((B * N, H * 72), float("nan"), dtype=torch.bfloat16, device=DEV)
        lse = torch.full((B, H, N), float("nan"), dtype=torch.float32, device=DEV) if with_lse else None
        lib.flash_attn(q, k, v, out, B=B, H=H, Nq=N, Nk=N, kv_rows=B * N, kv_len=lens, q_strides=(H * 72, 72),
                       k_strides=(H * 72, 72), v_strides=(H * 72, 72), lse=lse, fp32_p=fp32_p, reverse_batch=rev)
        outs.append(out)
        lses.append(lse)
    assert torch.equal(outs[0], outs[1])
    if with_lse:
        assert torch.equal(lses[0], lses[1])


def test_flash_attn_ragged_key_sets_with_an_empty_one():
    """Ragged key sets -- odd and even numbers of key blocks, a partial last block, a single block, an EMPTY key set in the
    middle: the output is finite and the empty key set gives zeros."""
    B, H, N, Nk = 6, 16, 2048, 704
    q, kv = _randn(B * N, H * 72, seed=130), _randn(B * Nk, 2 * H * 72, seed=131)
    lens = torch.tensor([704, 65, 0, 300, 128, 449], dtype=torch.int32, device=DEV)
    off = (torch.arange(B, device=DEV, dtype=torch.int32) * Nk).contiguous()
    out = torch.full((B * N, H * 72), float("nan"), dtype=torch.bfloat16, device=DEV)
    lse = torch.full((B, H, N), float("nan"), dtype=torch.float32, device=DEV)
    lib.flash_attn(q, kv[:, :H * 72], kv[:, H * 72:], out, B=B, H=H, Nq=N, Nk=Nk, kv_rows=B * Nk, kv_len=lens, kv_off=off,
                   q_strides=(H * 72, 72), k_strides=(2 * H * 72, 72), v_strides=(2 * H * 72, 72), lse=lse)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and (out.view(B, N, -1)[2] == 0).all()


@pytest.mark.parametrize("rev", [False, True])
def test_flash_attn_fp32_p_mode_matches_fp32_attention(rev):
    """`fp32_attention` (PixArt_blocks.py:145-147: q / k / v -- and therefore P -- kept in fp32 through P V): p_precision = 1
    feeds P to the tensor pipe as bf16 hi + lo terms.  Against the fp32 attention of the same bf16 q / k / v the result is then
    the CORRECTLY ROUNDED bf16 output for nearly every element (the only error left is the final bf16 store), while the default
    mode (P rounded to bf16, up to 2^-8) misses the correctly rounded value much more often.  Ragged key sets incl. a partial last
    sub-block, a single sub-block and an empty set; 4 work items per CTA under the persistent grid at the larger size."""
    for (B, H, N, Nk, lens) in [(2, 3, 300, 300, [300, 77]), (5, 16, 2048, 1024, [1024, 65, 0, 449, 1000])]:
        q, k, v = _randn(B, N, H, 72, seed=140), _randn(B, Nk, H, 72, seed=141), _randn(B, Nk, H, 72, seed=142)
        kl = torch.tensor(lens, dtype=torch.int32, device=DEV)
        want = torch.zeros(B, N, H, 72, dtype=torch.float64, device=DEV)     # float64: the check below is about single ulps of bf16
        for b, L in enumerate(lens):
            if L:
                sc = torch.einsum("nhd,mhd->hnm", q[b].double(), k[b, :L].double()) * 72 ** -0.5
                want[b] = torch.einsum("hnm,mhd->nhd", torch.softmax(sc, -1), v[b, :L].double())
        want = want.reshape(B * N, H * 72).float()
        outs, lses = {}, {}
        for fp32_p in (False, True):
            out = torch.full((B * N, H * 72), float("nan"), dtype=torch.bfloat16, device=DEV)
            lse = torch.full((B, H, N), float("nan"), dtype=torch.float32, device=DEV)
            lib.flash_attn(q, k, v, out, B=B, H=H, Nq=N, Nk=Nk, kv_rows=B * Nk, kv_len=kl, q_strides=(H * 72, 72),
                           k_strides=(H * 72, 72), v_strides=(H * 72, 72), lse=lse, fp32_p=fp32_p,
                           reverse_batch=rev)
            outs[fp32_p], lses[fp32_p] = out, lse
        torch.cuda.synchronize()
        assert torch.isfinite(outs[True].float()).all()
        assert torch.equal(lses[True], lses[False])                 # same fp32 logits and statistics in both modes
        e_split, e_bf16 = po.rel_err(outs[True].float(), want), po.rel_err(outs[False].float(), want)
        rounded = want.to(torch.bfloat16)
        miss_split = (outs[True] != rounded).float().mean().item()
        miss_bf16 = (outs[False] != rounded).float().mean().item()
        print(f"fp32_p B={B} N={N} Nk={Nk}: rel_err split {e_split:.3e} / bf16-P {e_bf16:.3e}; "
              f"not correctly rounded: split {miss_split:.4f} / bf16-P {miss_bf16:.4f}")
        assert e_split < 2.5e-3 and e_split <= e_bf16 * 1.001       # 2^-9 / sqrt(3) = 1.1e-3 is the bf16 store alone
        assert miss_split < 0.05 and miss_split < 0.25 * miss_bf16
