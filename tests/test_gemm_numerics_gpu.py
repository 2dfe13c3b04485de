"""The wgmma GEMM family (-m gpu) element by element against float64, on real (non-integer) data at the model's shapes
(XL/2: C = 1152, MLP 4608, 2048 image rows = B = 2 at 512 px, 600 caption rows, unless noted): every epilogue of pxa_gemm_bf16, the LoRA down-projection
and K-tail, the split-K weight gradient, the 3x3 convolution and the fused LayerNorm chain.  The bounds
and their derivation are in gemm_bounds.py; test_gemm_numerics_cpu.py shows they are attainable and reject the defects they
are meant to catch.

Inputs are read through row strides whose padding is NaN, and outputs are written into wider sentinel-filled buffers whose
guard band must come back unchanged.  With -s every check prints its largest err / bound and its bias statistic.
"""
import pytest
import torch

import gemm_bounds as gb

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
DEV = "cuda"
BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
C, HID = 1152, 4608
M_IMG = 2 * 1024                    # B = 2 samples of 32 x 32 tokens (the 512 px grid; 1024 px has 4096 per sample)


def rnd(*shape, seed, scale=1.0, dtype=BF):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV, dtype=F32) * scale).to(dtype)


def d(t):
    return None if t is None else t.double()


def gemm(a, w, bias, N, *, out_dtype=BF, epilogue=None, residual=None, aux=False, pre=None, tail=None, **kw):
    """lib.gemm on NaN-padded operands into a sentinel-banded output (residual: its fp32 / bf16 values copied in first).
    Returns out, aux (or None) as float64 after checking the guard bands."""
    M = a.shape[0]
    out, obuf = gb.sentinel_out(M, N, out_dtype, DEV, fill=residual)
    auxv = abuf = None
    if aux:
        auxv, abuf = gb.sentinel_out(M, N, BF, DEV)
    prev = pbuf = None
    if pre is not None:
        prev, pbuf = gb.sentinel_out(M, N, BF, DEV, fill=pre)
    if epilogue is None:
        epilogue = lib.EPI_BIAS_RESIDUAL if residual is not None else lib.EPI_BIAS
    res = out if residual is not None else prev
    ta = tw = None
    if tail is not None:
        ta, tw = gb.nan_padded(tail[0]), gb.nan_padded(tail[1])
    lib.gemm(gb.nan_padded(a), gb.nan_padded(w), bias, out, epilogue=epilogue, residual=res, out_aux=auxv, tail_a=ta,
             tail_w=tw, **kw)
    torch.cuda.synchronize()
    gb.assert_guard(obuf, M, N, "out")
    if abuf is not None:
        gb.assert_guard(abuf, M, N, "aux")
    if pbuf is not None:
        gb.assert_guard(pbuf, M, N, "pre")
    return out.double(), (auxv.double() if aux else None)


def acc_of(a, w, tail=None):
    if tail is not None:
        return gb.accumulate(*gb.with_tail(a.double(), w.double(), tail[0].double(), tail[1].double()))[:2]
    return gb.accumulate(a.double(), w.double())[:2]


def gates(M, N, rpb, seed, scale=1.0):
    """A per-sample fp32 gate read through a (samples, 2 N) buffer at column N (gate_batch_stride 2 N), and its per-row
    float64 expansion."""
    ns = -(-M // rpb)
    buf = rnd(ns, 2 * N, seed=seed, scale=scale, dtype=F32)
    g = buf[:, N:]
    return g, g.double().repeat_interleave(rpb, 0)[:M]


# ------------------------------------------------------------------------------------------------- forward projections
FWD = {
    # name: (M, K, N, weight scale, epilogue, block_n, extra kwargs)
    "qkv": (M_IMG, C, 3 * C, 1.0, "bias", 0, {}),
    "qkv_bn128": (M_IMG, C, 3 * C, 1.0, "bias", 128, {}),
    "qkv_bn192": (M_IMG, C, 3 * C, 1.0, "bias", 192, {}),
    "qkv_bn256": (M_IMG, C, 3 * C, 1.0, "bias", 256, {}),
    "qkv_reverse_tiles": (M_IMG, C, 3 * C, 1.0, "bias", 0, dict(reverse_tiles=True)),
    "qkv_max_ctas3": (M_IMG, C, 3 * C, 1.0, "bias", 0, dict(max_ctas=3)),
    "cross_q": (M_IMG, C, C, 1.0, "bias", 0, {}),
    "cross_kv": (600, C, 2 * C, 1.0, "bias", 0, {}),
    "cross_kv_stacked": (600, C, 28 * 2 * C, 1.0, "bias", 0, {}),
    "fc1_gelu": (M_IMG, C, HID, 3.0, "gelu", 0, {}),
    "fc2": (M_IMG, HID, C, 1.0, "bias", 0, {}),
    "y_proj_fc1_gelu": (600, 4096, C, 1.0, "gelu", 0, {}),
    "y_proj_fc2": (600, C, C, 1.0, "bias", 0, {}),
}


@pytest.mark.parametrize("name", list(FWD))
def test_forward_projection(name):
    M, K, N, ws, epi, bn, kw = FWD[name]
    a, w = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=ws * K ** -0.5)
    bias = rnd(N, seed=3, scale=0.1)
    ep = lib.EPI_BIAS_GELU if epi == "gelu" else lib.EPI_BIAS
    got, _ = gemm(a, w, bias, N, epilogue=ep, block_n=bn, **kw)
    acc, s = acc_of(a, w)
    y, sy = gb.bias_out(acc, s, d(bias))
    if epi == "gelu":
        gb.Tally(f"{name} out", c=1.0, tiny=gb.GELU_TINY).add(got, *gb.gelu_out(y, sy)).check()
    else:
        gb.Tally(f"{name} out").add(got, y, sy).check()


RPBS = [1024, 333, 96]


@pytest.mark.parametrize("rpb", RPBS)
@pytest.mark.parametrize("proj", ["attn_proj", "fc2"])
def test_gated_fp32_residual(proj, rpb):
    """attn proj / fc2 as the in-place fp32 gated residual x += gate[b] (A W^T + b); rows_per_batch 96 takes the per-row
    gate lookup (several samples per tile).  Also writes the bf16 copy of out (aux)."""
    K = C if proj == "attn_proj" else HID
    M, N = M_IMG, C
    a, w = rnd(M, K, seed=10), rnd(N, K, seed=11, scale=K ** -0.5)
    bias = rnd(N, seed=12, scale=0.1)
    x = rnd(M, N, seed=13, dtype=F32)
    g, gd = gates(M, N, rpb, seed=14)
    got, aux = gemm(a, w, bias, N, out_dtype=F32, residual=x, aux=True, gate=g, gate_batch_stride=2 * N, rows_per_batch=rpb)
    acc, s = acc_of(a, w)
    y, sy = gb.bias_out(acc, s, d(bias))
    o, so = gb.residual_out(y, sy, gd, d(x))
    gb.Tally(f"{proj} rpb {rpb} fp32 residual", fp32=True).add(got, o, so).check()
    gb.Tally(f"{proj} rpb {rpb} aux", tiny=0).add(aux, o, gb.f32_total(o, so)).check()


# ------------------------------------------------------------------------------------------------- training epilogues
def test_gelu_aux():
    M, K, N = M_IMG, C, HID
    a, w, bias = rnd(M, K, seed=20), rnd(N, K, seed=21, scale=3 * K ** -0.5), rnd(N, seed=22, scale=0.1)
    got, aux = gemm(a, w, bias, N, epilogue=lib.EPI_BIAS_GELU_AUX, aux=True)
    acc, s = acc_of(a, w)
    y, sy = gb.bias_out(acc, s, d(bias))
    gb.Tally("fc1 EPI_BIAS_GELU_AUX out", c=1.0, tiny=gb.GELU_TINY).add(got, *gb.gelu_out(y, sy)).check()
    gb.Tally("fc1 EPI_BIAS_GELU_AUX aux").add(aux, y, sy).check()


def test_mul_dgelu_fc2_dx():
    """fc2's dX = (dY W2) * gelu'(pre): dY (M, 1152), the transposed shadow W2^T (4608, 1152), N = 4608."""
    M, K, N = M_IMG, C, HID
    dy, w2t = rnd(M, K, seed=30), rnd(N, K, seed=31, scale=K ** -0.5)
    pre = rnd(M, N, seed=32, scale=3.0)
    got, _ = gemm(dy, w2t, None, N, epilogue=lib.EPI_MUL_DGELU, pre=pre)
    acc, s = acc_of(dy, w2t)
    gb.Tally("fc2 dX EPI_MUL_DGELU", tiny=gb.GELU_TINY).add(got, *gb.dgelu_out(acc, s, d(pre))).check()


@pytest.mark.parametrize("K,N", [(3 * C, C), (C, C), (HID, C)])
def test_dx_transposed_shadow(K, N):
    """dX = dY W through the transposed shadow W^T (K_in, N_out) as the GEMM weight: qkv (K = 3456), proj, fc2's input side."""
    dy, wt = rnd(M_IMG, K, seed=40), rnd(N, K, seed=41, scale=K ** -0.5)
    got, _ = gemm(dy, wt, None, N)
    acc, s = acc_of(dy, wt)
    gb.Tally(f"dX K={K}").add(got, acc, s).check()


@pytest.mark.parametrize("aux_is_branch", [False, True])
def test_bf16_residual_and_aux_branch(aux_is_branch):
    """The bf16 residual output (out = bf16(r + gate y)) and, with aux_is_branch, aux = the branch output y."""
    M, K, N = M_IMG, C, C
    a, w, bias = rnd(M, K, seed=50), rnd(N, K, seed=51, scale=K ** -0.5), rnd(N, seed=52, scale=0.1)
    r = rnd(M, N, seed=53)
    g, gd = gates(M, N, 1024, seed=54)
    got, aux = gemm(a, w, bias, N, residual=r, aux=True, gate=g, gate_batch_stride=2 * N, rows_per_batch=1024,
                    aux_is_branch=aux_is_branch)
    acc, s = acc_of(a, w)
    y, sy = gb.bias_out(acc, s, d(bias))
    o, so = gb.residual_out(y, sy, gd, d(r), bf16=True)
    gb.Tally("bf16 residual out").add(got, o, so).check()
    if aux_is_branch:
        gb.Tally("aux_is_branch aux").add(aux, y, sy).check()
    else:
        gb.Tally("bf16 residual aux").add(aux, o, so).check()


# ------------------------------------------------------------------------------------------------- LoRA
@pytest.mark.parametrize("rank", [8, 16, 24, 48, 96])
def test_lora_down_projection(rank):
    """u = x A^T: N = rank, narrower than one 32-column output slab for rank < 32."""
    a, w = rnd(M_IMG, C, seed=60), rnd(rank, C, seed=61, scale=C ** -0.5)
    got, _ = gemm(a, w, None, rank)
    acc, s = acc_of(a, w)
    gb.Tally(f"LoRA down rank {rank}").add(got, acc, s).check()


TAIL_EPIS = ["bias", "gelu", "gelu_aux", "mul_dgelu", "f32_residual", "bf16_residual"]


@pytest.mark.parametrize("epi", TAIL_EPIS)
@pytest.mark.parametrize("T", [8, 16, 24, 64, 72, 200])
def test_lora_tail(T, epi):
    """A W^T + tail_a tail_w^T under every epilogue; the fp32 residual tail runs at block_n 128."""
    M, K, N = 1024, C, C
    a, w = rnd(M, K, seed=70), rnd(N, K, seed=71, scale=(3.0 if "gelu" in epi else 1.0) * K ** -0.5)
    tail = (rnd(M, T, seed=72, scale=0.5), rnd(N, T, seed=73, scale=T ** -0.5))
    bias = None if epi == "mul_dgelu" else rnd(N, seed=74, scale=0.1)
    acc, s = acc_of(a, w, tail)
    y, sy = gb.bias_out(acc, s, d(bias))
    name = f"LoRA tail T={T} {epi}"
    if epi in ("bias", "gelu"):
        got, _ = gemm(a, w, bias, N, epilogue=lib.EPI_BIAS if epi == "bias" else lib.EPI_BIAS_GELU, tail=tail)
        if epi == "bias":
            gb.Tally(name).add(got, y, sy).check()
        else:
            gb.Tally(name, c=1.0, tiny=gb.GELU_TINY).add(got, *gb.gelu_out(y, sy)).check()
    elif epi == "gelu_aux":
        got, aux = gemm(a, w, bias, N, epilogue=lib.EPI_BIAS_GELU_AUX, aux=True, tail=tail)
        gb.Tally(name, c=1.0, tiny=gb.GELU_TINY).add(got, *gb.gelu_out(y, sy)).check()
        gb.Tally(name + " aux").add(aux, y, sy).check()
    elif epi == "mul_dgelu":
        pre = rnd(M, N, seed=75, scale=3.0)
        got, _ = gemm(a, w, None, N, epilogue=lib.EPI_MUL_DGELU, pre=pre, tail=tail)
        gb.Tally(name, tiny=gb.GELU_TINY).add(got, *gb.dgelu_out(acc, s, d(pre))).check()
    else:
        fp32 = epi == "f32_residual"
        r = rnd(M, N, seed=76, dtype=F32 if fp32 else BF)
        g, gd = gates(M, N, 512, seed=77)
        got, _ = gemm(a, w, bias, N, out_dtype=F32 if fp32 else BF, residual=r, gate=g, gate_batch_stride=2 * N,
                      rows_per_batch=512, tail=tail, block_n=128 if fp32 else 0)
        o, so = gb.residual_out(y, sy, gd, d(r), bf16=not fp32)
        gb.Tally(name, fp32=fp32).add(got, o, so).check()


def test_lora_tail_fused_qkv_block_diagonal():
    """The fused qkv tail: tail_a = [u_q | u_k | u_v] (M, 3 r), tail_w block-diagonal (3456, 3 r), one K-tail."""
    M, K, N, r = M_IMG, C, 3 * C, 16
    a, w, bias = rnd(M, K, seed=80), rnd(N, K, seed=81, scale=K ** -0.5), rnd(N, seed=82, scale=0.1)
    ta = rnd(M, 3 * r, seed=83, scale=0.5)
    tw = torch.zeros(N, 3 * r, dtype=BF, device=DEV)
    for i in range(3):
        tw[i * C:(i + 1) * C, i * r:(i + 1) * r] = rnd(C, r, seed=84 + i, scale=r ** -0.5)
    got, _ = gemm(a, w, bias, N, tail=(ta, tw))
    acc, s = acc_of(a, w, (ta, tw))
    y, sy = gb.bias_out(acc, s, d(bias))
    gb.Tally("LoRA fused-qkv block-diagonal tail").add(got, y, sy).check()


# ------------------------------------------------------------------------------------------------- weight gradient
def auto_splits(M, N, K, max_ctas=0):
    """The split count launch_wgrad picks for k_splits = 0 (gemm_sm100.cu): the most even wave over the SMs."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if 0 < max_ctas < sms:
        sms = max_ctas
    return gb.auto_splits(M, N, K, sms)


def check_wgrad(a_t, w_t, k_splits, name):
    K, M = a_t.shape
    N = w_t.shape[1]
    bucket = rnd(M, N, seed=99, dtype=F32, scale=float(K) ** 0.5)
    out, buf = gb.sentinel_out(M, N, F32, DEV, fill=bucket)
    lib.gemm_wgrad(gb.nan_padded(a_t), gb.nan_padded(w_t), out, k_splits=k_splits)
    torch.cuda.synchronize()
    gb.assert_guard(buf, M, N, "out")
    ks = k_splits or auto_splits(M, N, K)
    acc, s, parts = gb.accumulate(a_t.T.double(), w_t.T.double(), k_splits=ks)
    parts = acc.abs() if parts is None else parts
    gb.Tally(f"{name} (k_splits {ks})", fp32=True).add(out, d(bucket) + acc, s + ks * gb.U * (d(bucket).abs() + parts)).check()


@pytest.mark.parametrize("k_splits", [1, 2, 3, 4, 5, 0])
@pytest.mark.parametrize("rows", [2048, 8192])
def test_wgrad(rows, k_splits):
    """dW (1152, 1152) += dY^T X over `rows` token rows, onto a non-zero fp32 bucket."""
    dy, x = rnd(rows, C, seed=90), rnd(rows, C, seed=91)
    check_wgrad(dy, x, k_splits, f"wgrad rows {rows}")


@pytest.mark.parametrize("rank", [8, 16, 48, 96])
def test_wgrad_lora(rank):
    """The LoRA weight gradients: dA (rank, 1152) = (dY B)^T X (M = rank) and dB (1152, rank) = dY^T u (N = rank)."""
    rows = 2048
    t, x, dy = rnd(rows, rank, seed=92), rnd(rows, C, seed=93), rnd(rows, C, seed=94)
    check_wgrad(t, x, 0, f"wgrad LoRA dA rank {rank}")
    check_wgrad(dy, t, 0, f"wgrad LoRA dB rank {rank}")


# ------------------------------------------------------------------------------------------------- 3x3 convolution
CONV = [
    # (B, H, W, Cin, Cout, residual): decoder stages of the 1024 px VAE (latent 128) and a virtual-width aspect bucket
    (1, 128, 128, 512, 512, False),
    (1, 128, 128, 512, 512, True),
    (1, 256, 256, 512, 256, False),
    (1, 256, 256, 256, 256, True),
    (1, 512, 512, 256, 128, False),
    (1, 512, 512, 128, 128, True),
    (2, 104, 152, 512, 512, True),
    (2, 32, 32, 128, 128, False),
]


@pytest.mark.parametrize("geom", CONV, ids=lambda g: "x".join(map(str, g[:5])) + ("_res" if g[5] else ""))
def test_conv3x3(geom):
    Bc, H, W, Cin, Cout, has_res = geom
    x = rnd(Bc, H, W, Cin, seed=100)
    w = rnd(Cout, 3, 3, Cin, seed=101, scale=(9 * Cin) ** -0.5)
    bias = rnd(Cout, seed=102, scale=0.1)
    res = rnd(Bc, H, W, Cout, seed=103) if has_res else None
    out = torch.full((Bc, H, W, Cout), gb.SENTINEL, dtype=BF, device=DEV)
    lib.conv3x3_nhwc(x, w, bias, out, residual=res)
    torch.cuda.synchronize()
    acc, s = gb.conv_accumulate(x.double(), w.double())
    y, sy = gb.bias_out(acc, s, d(bias))
    name = f"conv3x3 {Bc}x{H}x{W} {Cin}->{Cout}"
    got = out.reshape(-1, Cout).double()
    if has_res:
        o, so = gb.residual_out(y, sy, torch.ones_like(y), d(res).reshape(-1, Cout), bf16=True)
        gb.Tally(name + " residual").add(got, o, so).check()
    else:
        gb.Tally(name).add(got, y, sy).check()


# ------------------------------------------------------------------------------------------------- fused LayerNorm chain
def offset_rows(M, ratio, seed):
    """fp32 rows with |mean| / std = ratio (per-row mean of random sign)."""
    x = rnd(M, C, seed=seed, dtype=F32)
    sgn = torch.sign(rnd(M, 1, seed=seed + 1, dtype=F32))
    return x + ratio * sgn


@pytest.mark.parametrize("ratio", [0, 4, 32])
def test_ln_prepare(ratio):
    M, rpb = M_IMG, 1024
    x = offset_rows(M, ratio, seed=110)
    mult = (1 + 0.3 * rnd(2, C, seed=112, dtype=F32)).contiguous()
    a = torch.empty(M, C, dtype=BF, device=DEV)
    stats = torch.full((M, lib.LN_STAT_PARTS, 2), float("nan"), device=DEV)
    xp = gb.nan_padded(x)
    lib.ln_prepare(xp, mult, a, stats, mod_batch_stride=C, rows_per_batch=rpb)
    torch.cuda.synchronize()
    ref, s, st, s_st = gb.ln_prepare_ref(d(x), mult.double().repeat_interleave(rpb, 0))
    gb.Tally(f"ln_prepare a, mean/std {ratio}").add(a.double(), ref, s).check()
    gb.Tally(f"ln_prepare stats, mean/std {ratio}", fp32=True).add(stats[:, 0].double(), st, s_st).check()
    assert (stats[:, 1:] == 0).all()


def test_ln_skinny_hi_lo():
    """The skinny GEMM of the fused-LN conditioning: bf16 hi / lo rows of a few fp32 rows, accumulated in place onto a zeroed
    fp32 buffer (EPI_BIAS_RESIDUAL, no gate) against the stacked qkv | fc1 weights of two blocks."""
    rows = rnd(8, C, seed=120, dtype=F32) * 0.2
    hi = rows.to(BF)
    lo = (rows - hi.float()).to(BF)
    a = torch.cat([hi, lo]).contiguous()
    N = 2 * (3 * C + HID)
    w = rnd(N, C, seed=121, scale=C ** -0.5)
    got, _ = gemm(a, w, None, N, out_dtype=F32, residual=torch.zeros(16, N, device=DEV))
    acc, s = acc_of(a, w)
    gb.Tally("LN skinny hi + lo", fp32=True).add(got, acc, s).check()


@pytest.mark.parametrize("bn,N", [(192, C), (192, 1088), (128, 1024)])
def test_residual_aux_scale_row_stats(bn, N):
    """The producer side of the fused LN chain: x += gate (A W^T + b), aux = bf16(x * aux_scale[b]) and the per-tile row
    statistics of x.  (192, 1088): a partial last column tile; (128, 1024): all 8 parts in use."""
    M, K, rpb = M_IMG, C, 1024
    a, w, bias = rnd(M, K, seed=130), rnd(N, K, seed=131, scale=K ** -0.5), rnd(N, seed=132, scale=0.1)
    x = rnd(M, N, seed=133, dtype=F32)
    g, gd = gates(M, N, rpb, seed=134, scale=0.3)
    sc = (1 + 0.3 * rnd(2, N, seed=135, dtype=F32)).contiguous()
    stats = torch.full((M, lib.LN_STAT_PARTS, 2), float("nan"), device=DEV)
    got, aux = gemm(a, w, bias, N, out_dtype=F32, residual=x, aux=True, gate=g, gate_batch_stride=2 * N, rows_per_batch=rpb,
                    aux_scale=sc, aux_scale_batch_stride=N, row_stats_out=stats, block_n=bn)
    acc, s = acc_of(a, w)
    y, sy = gb.bias_out(acc, s, d(bias))
    o, so = gb.residual_out(y, sy, gd, d(x))
    gb.Tally(f"LN producer bn {bn} N {N} out", fp32=True).add(got, o, so).check()
    scd = sc.double().repeat_interleave(rpb, 0)
    gb.Tally(f"LN producer bn {bn} N {N} aux_scale").add(aux, *gb.aux_out(o, gb.f32_total(o, so), scd)).check()
    ref, slack, parts = gb.row_stats_ref(got, bn)
    gb.Tally(f"LN producer bn {bn} N {N} row_stats", fp32=True).add(stats[:, :parts].double(), ref, slack).check()
    assert (stats[:, parts:] == 0).all(), "row_stats_out: unused parts not zeroed"


def test_row_stats_too_many_parts_rejected():
    """N = 1152 at block_n 128 needs 9 column tiles, one more than PXA_LN_STAT_PARTS: PXA_ERR_ARG, nothing written."""
    M, N = 256, C
    a, w = rnd(M, C, seed=140), rnd(N, C, seed=141, scale=C ** -0.5)
    x = rnd(M, N, seed=142, dtype=F32)
    before = x.clone()
    stats = torch.zeros(M, lib.LN_STAT_PARTS, 2, device=DEV)
    with pytest.raises(lib.PxaError, match="PXA_LN_STAT_PARTS"):
        lib.gemm(a, w, None, x, epilogue=lib.EPI_BIAS_RESIDUAL, residual=x, row_stats_out=stats, block_n=128)
    torch.cuda.synchronize()
    assert torch.equal(x, before)


@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("ratio", [0, 1, 4, 32])
def test_ln_epilogue_formula(ratio, gelu):
    """EPI_LN_BIAS / EPI_LN_BIAS_GELU against the kernel's formula rstd (acc - mu u_b) + v_b, with a and the statistics
    from pxa_ln_prepare at |mean| / std = ratio."""
    M, rpb, N = M_IMG, 1024, 3 * C if not gelu else HID
    x = offset_rows(M, ratio, seed=150)
    mult = (1 + 0.3 * rnd(2, C, seed=152, dtype=F32)).contiguous()
    a = torch.empty(M, C, dtype=BF, device=DEV)
    stats = torch.empty(M, lib.LN_STAT_PARTS, 2, device=DEV)
    lib.ln_prepare(x, mult, a, stats, mod_batch_stride=C, rows_per_batch=rpb)
    w = rnd(N, C, seed=153, scale=(3.0 if gelu else 1.0) * C ** -0.5)
    u = rnd(2, N, seed=154, dtype=F32, scale=3.0)
    v = rnd(2, N, seed=155, dtype=F32)
    ep = lib.EPI_LN_BIAS_GELU if gelu else lib.EPI_LN_BIAS
    got, _ = gemm(a, w, None, N, epilogue=ep, rows_per_batch=rpb, ln_stats=stats, ln_u=u, ln_v=v, ln_uv_batch_stride=N,
                  ln_dim=C, ln_eps=1e-6)
    acc, s = acc_of(a, w)
    ud, vd = u.double().repeat_interleave(rpb, 0), v.double().repeat_interleave(rpb, 0)
    xr, sx = gb.ln_epilogue_ref(acc, s, stats.double(), ud, vd, C, 1e-6)
    name = f"EPI_LN_BIAS{'_GELU' if gelu else ''} mean/std {ratio}"
    if gelu:
        gb.Tally(name, c=1.0, tiny=gb.GELU_TINY).add(got, *gb.gelu_out(xr, sx)).check()
    else:
        gb.Tally(name).add(got, xr, sx).check()
