"""Element-wise numerics of the training-backward kernels (-m gpu) against float64 references on the same inputs, in the
style of test_numerics_gpu.py (whose helpers are reused):

- Exact constructions (`torch.equal`): integer inputs for which every product and every partial sum the kernel forms is
  representable, in any order of summation, so a single wrong, missing or doubled element fails.  Each docstring says why
  exactness holds.
- Guard bands: outputs are written into views at the front of, or column slices of, sentinel-filled buffers, which must come
  back bit-unchanged; inputs are read through slices whose padding is NaN.
- Element-wise contracts (`assert_bf16_close` / `assert_f32_close`): for the LayerNorm backward of ln_modulate_bwd and of the
  conv + LayerNorm KV compression, with slack derived from the kernel's summation structure (stated per test).

The shapes put sample boundaries inside the kernels' row blocks (32 rows per CTA in gate_residual_bwd, 16 rows per warp in
ln_modulate_bwd, 4 output tokens per warp / 32 per CTA in kv_compress_bwd, 128-row slabs in colsum) and leave tail warps,
tail CTAs and idle threads.  With -s every contract prints its largest error / bound.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from test_numerics_gpu import LOG2E, SENTINEL, _assert_pad_unchanged, _ints, _ln_slack, _offset_input, _one_key_problem, _padded, \
    _randn, assert_bf16_close, bf16_ulp

from norm_bounds import ln_bwd_slack as _ln_bwd_slack, ln_stats as _ln_stats, sample_sum_slack as _sample_sum_slack

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
DEV = "cuda"
U = 2.0 ** -24                      # fp32 unit roundoff


def f32_ulp(ref: torch.Tensor) -> torch.Tensor:
    """The spacing of fp32 numbers at |ref| (float64): 2^(e - 24) for |ref| in [2^(e-1), 2^e), 2^-149 below the normals."""
    _, e = torch.frexp(ref.abs())
    return torch.ldexp(torch.ones_like(ref), (e - 24).clamp(min=-149))


def assert_f32_close(got: torch.Tensor, ref: torch.Tensor, slack, *, name: str, max_ulp: float = 1.0) -> None:
    """fp32 counterpart of assert_bf16_close: |got - ref| <= max_ulp * ulp_fp32(ref) + slack element-wise, every result
    finite.  Prints the largest error / bound."""
    got, ref = got.double(), ref.double()
    slack = torch.zeros_like(ref) if slack is None else torch.as_tensor(slack, dtype=torch.float64, device=ref.device).expand_as(ref)
    got, ref, slack = got.flatten(), ref.flatten(), slack.flatten()
    assert torch.isfinite(got).all(), f"{name}: {(~torch.isfinite(got)).sum().item()} non-finite results"
    err = (got - ref).abs()
    bound = max_ulp * f32_ulp(ref) + slack
    ratio = (err / bound).max().item()
    print(f"{name}: {ref.numel()} elements, max |err| {err.max().item():.3e}, max err / bound {ratio:.3f}")
    bad = err > bound
    if bad.any():
        i = torch.nonzero(bad)[:5, 0]
        raise AssertionError(f"{name}: {bad.sum().item()} elements outside the bound, e.g. got {got[i].tolist()} want "
                             f"{ref[i].tolist()} bound {bound[i].tolist()}")


def _ratio(got, ref, slack, name):
    """Print the largest |got - ref| / (1 bf16 ulp + slack) of a bf16 output (assert_bf16_close asserts it)."""
    r = ((got.double() - ref).abs() / (bf16_ulp(ref) + slack)).max().item()
    print(f"{name}: max err / bound {r:.3f}")


def _front(rows, cols, fill, dtype, extra=3):
    """A contiguous (rows, cols) view at the front of a (rows + extra, cols) buffer filled with `fill`."""
    buf = torch.full((rows + extra, cols), fill, dtype=dtype, device=DEV)
    return buf[:rows], buf


# ------------------------------------------------------------------------------------------------- gate + residual
@pytest.mark.parametrize("C", [4, 72, 1152])
@pytest.mark.parametrize("M", [33, 1000, 4097])
@pytest.mark.parametrize("rpb", [1, 7, 31, 32, 33, 255, 0])
def test_gate_residual_exact(rpb, M, C):
    """gate_residual_bwd (dy = bf16(dout gate[b]), dgate[b] += sum_rows dout y) and gate_residual_fwd as BlockFn uses it
    (out = x + gate[b] y on the fp32 stream, and with gate None the fp32 + bf16 add of the residual-stream gradient).
    rows_per_batch 0 stands for M (one sample).  Exact: dout is an integer in [-64, 64] and gates are +-0.5, 1, 2, 4, so
    dout gate has at most 6 significant bits (bf16-exact); dout y with y in [-8, 8] is an integer, and every partial sum of
    dgate (a pre-filled integer plus <= 4097 terms of magnitude <= 512) is an integer below 2^24, exact in any order.  The
    forward sums are halves below 2^12, exact.  The CTA of gate_residual_bwd spans 32 rows and flushes dgate where the sample
    changes inside it; C = 4 / 72 leave 287 / 270 of its 288 threads idle.  dy / out / dgate are views at the front of
    sentinel-filled buffers; with dgate None, y is NaN-filled and must not be read."""
    rpb = rpb or M
    B = (M + rpb - 1) // rpb
    g = torch.Generator().manual_seed(M * 7 + C + rpb)
    pick = torch.tensor([0.5, -0.5, 1.0, 2.0, 4.0])
    mod = torch.full((B, 6, C), float("nan"), dtype=torch.float32)
    mod[:, 2] = pick[torch.randint(0, len(pick), (B, C), generator=g)]
    mod = mod.to(DEV)
    gate = mod[:, 2]
    b_of = torch.arange(M, device=DEV) // rpb
    grow = gate.double()[b_of]
    dout = _ints(M, C, lo=-64, hi=64, seed=M + C, dtype=torch.float32)
    y = _ints(M, C, lo=-8, hi=8, seed=M + C + 1)
    dy, dybuf = _front(M, C, SENTINEL, torch.bfloat16)
    dgate, dgbuf = _front(B, C, SENTINEL, torch.float32)
    dgate.copy_(_ints(B, C, lo=-1000, hi=1000, seed=M + C + 2, dtype=torch.float32))
    want_dg = dgate.double().index_add(0, b_of, dout.double() * y.double())
    before, dgbefore = dybuf.clone(), dgbuf.clone()
    lib.gate_residual_bwd(dout, y, gate, dy, dgate, gate_batch_stride=mod.stride(0), rows_per_batch=rpb)
    assert torch.equal(dy.double(), dout.double() * grow), "dy"
    assert torch.equal(dgate.double(), want_dg), "dgate"
    assert torch.equal(dybuf[M:], before[M:]) and torch.equal(dgbuf[B:], dgbefore[B:]), "rows past dy / dgate were written"
    nan_y = torch.full_like(y, float("nan"))
    for gt in (gate, None):                          # no gate gradient: y is not read
        dy.fill_(SENTINEL)
        lib.gate_residual_bwd(dout, nan_y, gt, dy, None, gate_batch_stride=mod.stride(0), rows_per_batch=rpb)
        assert torch.equal(dy.double(), dout.double() * (grow if gt is not None else 1.0)), f"dy, gate={gt is not None}"
        assert torch.equal(dybuf[M:], before[M:])
    x = _ints(M, C, lo=-512, hi=512, seed=M + C + 3, dtype=torch.float32) * 0.5
    out, obuf = _front(M, C, SENTINEL, torch.float32)
    obefore = obuf.clone()
    for gt in (gate, None):
        lib.gate_residual_fwd(x, y, gt, out, gate_batch_stride=mod.stride(0), rows_per_batch=rpb)
        assert torch.equal(out.double(), x.double() + (grow if gt is not None else 1.0) * y.double()), f"fwd gate={gt is not None}"
        assert torch.equal(obuf[M:], obefore[M:])


# ------------------------------------------------------------------------------------------------- column sums
@pytest.mark.parametrize("N", [8, 248, 256, 264, 1152, 4608])
@pytest.mark.parametrize("M", [1, 7, 8, 24, 25, 32, 33, 127, 128, 129, 1000, 16385])
def test_colsum_exact(M, N):
    """colsum: out[c] += sum_r a[r, c].  a holds integers in [-8, 8], out a pre-filled integer, so every partial sum (per
    row lane, in shared memory, and the per-CTA fp32 atomics) is an integer below 2^24: exact in any order.  M covers the
    128-row slab tails and the remainder of the 4-loads-in-flight loop (rows lane + 32 k, stopping once r + 24 >= the slab
    end); N = 8 / 248 / 264 leave 31 / 1 / 31 idle column threads of a CTA.  a is a column slice of a buffer whose 8 + 16
    padding columns are NaN; out sits at the front of a sentinel buffer."""
    abuf = torch.full((M, N + 24), float("nan"), dtype=torch.bfloat16, device=DEV)
    a = abuf[:, 8:8 + N]
    a.copy_(_ints(M, N, lo=-8, hi=8, seed=M * 31 + N))
    obuf = torch.full((N + 13,), SENTINEL, dtype=torch.float32, device=DEV)
    out = obuf[:N]
    out.copy_(_ints(N, lo=-100, hi=100, seed=M + N, dtype=torch.float32))
    want = out.double() + a.double().sum(0)
    before = obuf.clone()
    lib.colsum(a, out)
    assert torch.equal(out.double(), want)
    assert torch.equal(obuf[N:], before[N:]), "entries past out were written"


# ------------------------------------------------------------------------------------------------- attention delta
@pytest.mark.parametrize("Nq", [1, 5, 201])
@pytest.mark.parametrize("H", [1, 3, 16])
def test_attn_delta_exact(H, Nq):
    """delta[(b H + h) Nq + i] = sum_d dO[b, i, h, d] o[b, i, h, d], read back through flash_attn_bwd(delta=buf).  o and dO
    are integers in [-4, 4], so each of the 72 products is an integer <= 16 and every partial sum is an integer <= 1152:
    exact.  B = 2: B Nq H is never a multiple of the 256-thread CTA.  o / dO have row stride H 72 + 8 and NaN padding
    columns; delta sits at the front of a sentinel buffer.  (q = k = 0 and lse = 0 keep the rest of the backward finite.)"""
    B, D, Nk = 2, 72, 64
    C = H * D
    o, _ = _padded(B * Nq, C, 8, float("nan"), torch.bfloat16)
    do, _ = _padded(B * Nq, C, 8, float("nan"), torch.bfloat16)
    o.copy_(_ints(B * Nq, C, lo=-4, hi=4, seed=H * 10 + Nq))
    do.copy_(_ints(B * Nq, C, lo=-4, hi=4, seed=H * 10 + Nq + 1))
    q = torch.zeros(B * Nq, C, dtype=torch.bfloat16, device=DEV)
    k = torch.zeros(B * Nk, C, dtype=torch.bfloat16, device=DEV)
    v = _ints(B * Nk, C, lo=-4, hi=4, seed=3)
    lse = torch.zeros(B, H, Nq, dtype=torch.float32, device=DEV)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    n = B * H * Nq
    dbuf = torch.full((n + 7,), SENTINEL, dtype=torch.float32, device=DEV)
    st = (C, D)
    lib.flash_attn_bwd(q, k, v, o, do, lse, dq, dk, dv, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=B * Nk, q_strides=st, k_strides=st,
                       v_strides=st, dq_strides=st, dk_strides=st, dv_strides=st, delta=dbuf[:n])
    want = (o.double() * do.double()).view(B, Nq, H, D).sum(-1).permute(0, 2, 1).reshape(-1)
    assert torch.equal(dbuf[:n].double(), want)
    assert (dbuf[n:] == SENTINEL).all(), "entries past delta were written"


# ------------------------------------------------------------------------------------------------- LN-modulate backward
@pytest.mark.parametrize("mode", ["distinct", "aliased"])
def test_ln_modulate_bwd_zero_gradient_passes_add_in_through(mode):
    """dxn = 0: every term of the norm's gradient is an exact (signed) zero, so dx = add_in + 0 must equal add_in bit for
    bit, also when add_in is dx itself (each element is read before the same thread writes it); dshift / dscale gain
    exact zeros and keep their pre-filled values.  M = 1001 rows over samples of 333."""
    M, C, rpb = 1001, 1152, 333
    B = (M + rpb - 1) // rpb
    x = _offset_input((M, C), 4, seed=70).float()
    mod = _randn(B, 6, C, seed=71, dtype=torch.float32) * 0.3
    dxn = torch.zeros(M, C, dtype=torch.bfloat16, device=DEV)
    add = _randn(M, C, seed=72, dtype=torch.float32)
    dsh, dsc = _randn(B, C, seed=73, dtype=torch.float32), _randn(B, C, seed=74, dtype=torch.float32)
    sh0, sc0 = dsh.clone(), dsc.clone()
    if mode == "aliased":
        dx = add.clone()
        lib.ln_modulate_bwd(x, dxn, mod[:, 1], dx, dsh, dsc, mod_batch_stride=mod.stride(0), rows_per_batch=rpb, add_in=dx)
    else:
        dx = torch.full_like(x, float("nan"))
        lib.ln_modulate_bwd(x, dxn, mod[:, 1], dx, dsh, dsc, mod_batch_stride=mod.stride(0), rows_per_batch=rpb, add_in=add)
    assert torch.equal(dx, add)
    assert torch.equal(dsh, sh0) and torch.equal(dsc, sc0)


def _ln_bwd_reference(x, dxn, scale_rows, eps):
    """float64 (xh, rstd, r, g, dx without add_in) of the LN-modulate backward; scale_rows (M, C) = scale[b(row)]."""
    xh, rstd, r = _ln_stats(x.double(), eps)
    g = dxn.double() * (1 + scale_rows)
    dx = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    return xh, rstd, r, g, dx


@pytest.mark.parametrize("eps", [1e-6, 1e-5])
@pytest.mark.parametrize("rpb", [1, 15, 16, 17, 255, 333])
@pytest.mark.parametrize("ratio", [0, 4, 32, 128])
def test_ln_modulate_bwd_elementwise(ratio, rpb, eps):
    """ln_modulate_bwd against the float64 LN-modulate backward on the same fp32 x (bf16 values ratio + N(0, 1): |mean| / std
    = ratio) and bf16 dxn, M = 1001 rows (not a multiple of 16 or 128; the last sample is partial), scale a strided column of
    a (B, 6, C) mod, for add_in absent, distinct and aliased (add_in is dx), dshift / dscale pre-filled.
    dx: 1 fp32 ulp (the add of add_in) + _ln_bwd_slack with rstd_rel = 2^-19 (the variance: 1152 squares in <= 41 fp32
    additions, then rsqrtf's 2 ulp: <= 23 u).  dshift: _sample_sum_slack of dxn (exact bf16 terms).  dscale: the same for the
    terms dxn xh (one fma each) plus sum |dxn| e for the error e of the kernel's xh (see _ln_bwd_slack)."""
    M, C = 1001, 1152
    B = (M + rpb - 1) // rpb
    x = _offset_input((M, C), ratio, seed=80 + ratio).float()
    mod = _randn(B, 6, C, seed=81, dtype=torch.float32) * 0.3
    dxn = _randn(M, C, seed=82 + rpb)
    b_of = torch.arange(M, device=DEV) // rpb
    xh, rstd, r, g, dx_core = _ln_bwd_reference(x, dxn, mod[:, 1].double()[b_of], eps)
    slack_dx = _ln_bwd_slack(xh, rstd, g, r, 2.0 ** -19)
    e = 2.0 ** -18 * (1 + r) + 2.0 ** -19 * xh.abs()
    for mode in ("none", "distinct", "aliased"):
        add = _randn(M, C, seed=83, dtype=torch.float32) * 2
        dsh, dsc = _randn(B, C, seed=84, dtype=torch.float32), _randn(B, C, seed=85, dtype=torch.float32)
        want_sh = dsh.double().index_add(0, b_of, dxn.double())
        want_sc = dsc.double().index_add(0, b_of, dxn.double() * xh)
        sl_sh = _sample_sum_slack(b_of, B, rpb, M, dxn.double(), dsh)
        sl_sc = _sample_sum_slack(b_of, B, rpb, M, dxn.double() * xh, dsc) + \
            torch.zeros_like(dsc, dtype=torch.float64).index_add(0, b_of, dxn.double().abs() * e)
        kw = dict(mod_batch_stride=mod.stride(0), rows_per_batch=rpb, eps=eps)
        if mode == "aliased":
            dx = add.clone()
            lib.ln_modulate_bwd(x, dxn, mod[:, 1], dx, dsh, dsc, add_in=dx, **kw)
        else:
            dx = torch.full_like(x, float("nan"))
            lib.ln_modulate_bwd(x, dxn, mod[:, 1], dx, dsh, dsc, add_in=add if mode == "distinct" else None, **kw)
        want_dx = dx_core + (add.double() if mode != "none" else 0.0)
        tag = f"ln_modulate_bwd mean/std={ratio} rpb={rpb} eps={eps:g} add_in={mode}"
        assert_f32_close(dx, want_dx, slack_dx, name=tag + " dx")
        assert_f32_close(dsh, want_sh, sl_sh, name=tag + " dshift")
        assert_f32_close(dsc, want_sc, sl_sc, name=tag + " dscale")


@pytest.mark.parametrize("ratio", [0, 32])
def test_ln_modulate_bwd_qk_norm_call_elementwise(ratio):
    """The qk_norm backward exactly as BlockFn calls it: M = 8192 rows, rows_per_batch = M (one "sample", so 512 warps
    flush their column sums into ONE row of dshift / dscale with fp32 atomics), scale = w - 1 of shape (1, C),
    mod_batch_stride = C, eps 1e-5; dshift / dscale are the gradients of the LayerNorm's bias / weight.  Same bounds as
    test_ln_modulate_bwd_elementwise (W_b = 512 atomics)."""
    M, C = 8192, 1152
    x = _offset_input((M, C), ratio, seed=90 + ratio).float()
    w = 1 + _randn(C, seed=91, scale=0.1, dtype=torch.float32)
    scale = (w - 1.0).view(1, C).contiguous()
    dxn = _randn(M, C, seed=92)
    b_of = torch.zeros(M, dtype=torch.long, device=DEV)
    xh, rstd, r, g, dx_core = _ln_bwd_reference(x, dxn, scale.double(), 1e-5)
    dsh, dsc = torch.zeros(1, C, device=DEV), torch.zeros(1, C, device=DEV)
    dx = torch.full_like(x, float("nan"))
    lib.ln_modulate_bwd(x, dxn, scale, dx, dsh, dsc, mod_batch_stride=C, rows_per_batch=M, eps=1e-5)
    e = 2.0 ** -18 * (1 + r) + 2.0 ** -19 * xh.abs()
    tag = f"ln_modulate_bwd qk_norm M={M} mean/std={ratio}"
    assert_f32_close(dx, dx_core, _ln_bwd_slack(xh, rstd, g, r, 2.0 ** -19), name=tag + " dx")
    assert_f32_close(dsh, dxn.double().sum(0, keepdim=True), _sample_sum_slack(b_of, 1, M, M, dxn.double(), dsh),
                     name=tag + " d bias")
    assert_f32_close(dsc, (dxn.double() * xh).sum(0, keepdim=True),
                     _sample_sum_slack(b_of, 1, M, M, dxn.double() * xh, dsc) + (dxn.double().abs() * e).sum(0, keepdim=True),
                     name=tag + " d weight")


# ------------------------------------------------------------------------------------------------- KV compression backward
@pytest.mark.parametrize("offset", [0, 32])
@pytest.mark.parametrize("B,H,W", [(2, 16, 16), (1, 16, 24), (3, 2, 2), (1, 6, 10), (2, 64, 64)])
def test_kv_compress_bwd_elementwise(B, H, W, offset):
    """kv_compress_bwd (depthwise 2x2 / s2 conv + bias, LayerNorm(affine, eps 1e-5), K and V) against float64 autograd of the
    same op on the same bf16 inputs and weights.  Inputs are offset + N(0, 1) per channel with taps 0.25 + 0.01 N(0, 1), so
    the conv output has |mean| / std up to ~40 over the channels (printed).  B H/2 W/2 = 128, 96, 3, 15, 2048 output tokens:
    tail warps (4 tokens each) and tail CTAs (32).  dqkv has row stride 3C + 64 (ld_din != ld_in), is sentinel-filled, and
    its Q slice and padding columns must come back bit-unchanged; the parameter gradients are pre-filled.
    Bounds, with da = rstd (g - mean g - xh mean(g xh)) the conv-output gradient (g = dy gamma):
      - da: _ln_bwd_slack with rstd_rel = 2^-19 (2 + r): besides the 23 u of the LN statistics, the 4 fp32 roundings of
        each conv output (4 u (|mean| + |s - mean|)) move the variance by <= 8 u (r + 4) relative;
      - d input = bf16(da w_t): 1 bf16 ulp + |w_t| slack(da);
      - parameter gradients: per CTA 32 rows of shared-memory atomics, then one global atomic per CTA (K and V CTAs alike,
        n_cta in all) onto the pre-filled value: (31 + n_cta) u (|pre| + sum|terms|), one u more where a term is a
        rounded product, plus the propagated error of the terms (sum |dy| e for d gamma, sum slack(da) |x_t| for d w)."""
    C = 1152
    Ho, Wo = H // 2, W // 2
    n_out, M = B * Ho * Wo, B * H * W
    n_cta = 2 * ((n_out + 31) // 32)
    gen = torch.Generator().manual_seed(B * 1000 + H * 10 + W + offset)
    qkv = ((torch.randn(M, 3 * C, generator=gen) + offset)).to(torch.bfloat16).to(DEV)
    conv_w = (0.25 + 0.01 * torch.randn(C, 1, 2, 2, generator=gen)).to(torch.bfloat16).to(DEV)
    conv_b = (0.1 * torch.randn(C, generator=gen)).to(torch.bfloat16).to(DEV)
    ln_w = (1 + 0.2 * torch.randn(C, generator=gen)).to(torch.bfloat16).to(DEV)
    ln_b = (0.1 * torch.randn(C, generator=gen)).to(torch.bfloat16).to(DEV)
    dkc = torch.randn(n_out, C, generator=gen).to(torch.bfloat16).to(DEV)
    dvc = torch.randn(n_out, C, generator=gen).to(torch.bfloat16).to(DEV)
    dbuf = torch.full((M, 3 * C + 64), SENTINEL, dtype=torch.bfloat16, device=DEV)
    pre = [torch.randn(s, generator=gen).to(DEV) for s in ((C, 1, 2, 2), (C,), (C,), (C,))]
    grads = [p.clone() for p in pre]
    before = dbuf.clone()
    lib.kv_compress_bwd(qkv[:, C:2 * C], qkv[:, 2 * C:], dkc, dvc, dbuf[:, C:2 * C], dbuf[:, 2 * C:3 * C], conv_w, conv_b, ln_w,
                        *grads, B=B, H=H, W=W, ld_in=3 * C, ld_din=dbuf.stride(0))
    # float64 reference (autograd) and the intermediates of the bounds
    f = qkv.double().requires_grad_(True)
    pw, pb, pg, pbeta = (t.double().requires_grad_(True) for t in (conv_w, conv_b, ln_w, ln_b))
    loss, inter = 0, []
    for i, d in ((1, dkc), (2, dvc)):
        img = f[:, i * C:(i + 1) * C].reshape(B, H, W, C).permute(0, 3, 1, 2)
        s = F.conv2d(img, pw, pb, stride=2, groups=C).reshape(B, C, -1).permute(0, 2, 1).reshape(n_out, C)
        loss = loss + (F.layer_norm(s, (C,), pg, pbeta, eps=1e-5) * d.double()).sum()
        inter.append(s.detach())
    loss.backward()
    s = torch.cat(inter)                                           # (2 n_out, C): K rows, then V rows
    dy = torch.cat([dkc, dvc]).double()
    xh, rstd, r = _ln_stats(s, 1e-5)
    g = dy * ln_w.double()
    mg, mgx = g.mean(-1, keepdim=True), (g * xh).mean(-1, keepdim=True)
    da = rstd * (g - mg - xh * mgx)
    sl_da = _ln_bwd_slack(xh, rstd, g, r, 2.0 ** -19 * (2 + r))
    e = 2.0 ** -18 * (1 + r) + 2.0 ** -19 * xh.abs()
    tag = f"kv_compress_bwd B={B} H={H} W={W} offset={offset} (conv out mean/std <= {r.max().item():.1f})"
    # input gradients: token (2 py + ty, 2 px + tx) of output (py, px) gets da w[tap]
    taps = conv_w.double().view(C, 4).T                            # (4, C), tap = 2 ty + tx
    sl_in = torch.zeros(2, B, H, W, C, dtype=torch.float64, device=DEV)
    sl6 = sl_da.view(2, B, Ho, Wo, C)
    for t in range(4):
        sl_in[:, :, t >> 1::2, t & 1::2] = sl6 * taps[t].abs()
    for i in (1, 2):
        got = dbuf[:, i * C:(i + 1) * C]
        slk = sl_in[i - 1].reshape(M, C)
        assert_bf16_close(got, f.grad[:, i * C:(i + 1) * C], slk, name=tag + (" dk_in", " dv_in")[i - 1])
        _ratio(got, f.grad[:, i * C:(i + 1) * C], slk, tag + (" dk_in", " dv_in")[i - 1])
    assert torch.equal(dbuf[:, :C], before[:, :C]), "the Q slice of dqkv was written"
    _assert_pad_unchanged(dbuf, 3 * C, before, "dqkv")
    # parameter gradients (K and V rows together)
    xin = torch.stack([torch.cat([f.detach()[:, i * C:(i + 1) * C].reshape(B, H, W, C)[:, t >> 1::2, t & 1::2].reshape(n_out, C)
                                  for i in (1, 2)]) for t in range(4)])            # (4, 2 n_out, C): x_t of each output row
    terms = ((da[None] * xin).sum(1).T, da.sum(0), (dy * xh).sum(0), dy.sum(0))
    for t_, ref in zip(terms, (pw.grad.view(C, 4), pb.grad, pg.grad, pbeta.grad)):    # the intermediates of the bounds
        assert torch.allclose(t_, ref, rtol=1e-9, atol=1e-9)                             # restate the autograd reference
    acc = lambda extra: (31 + extra + n_cta) * U
    p64 = [p.double() for p in pre]
    sl_w = acc(1) * (p64[0].view(C, 4).abs() + (da[None] * xin).abs().sum(1).T) + (sl_da[None] * xin.abs()).sum(1).T
    assert_f32_close(grads[0].view(C, 4), p64[0].view(C, 4) + pw.grad.view(C, 4), sl_w, name=tag + " d conv.weight")
    assert_f32_close(grads[1], p64[1] + pb.grad, acc(0) * (p64[1].abs() + da.abs().sum(0)) + sl_da.sum(0),
                     name=tag + " d conv.bias")
    assert_f32_close(grads[2], p64[2] + pg.grad, acc(1) * (p64[2].abs() + (dy * xh).abs().sum(0)) + (dy.abs() * e).sum(0),
                     name=tag + " d norm.weight")
    assert_f32_close(grads[3], p64[3] + pbeta.grad, acc(0) * (p64[3].abs() + dy.abs().sum(0)), name=tag + " d norm.bias")


# ------------------------------------------------------------------------------------------------- transpose, element-wise path
@pytest.mark.parametrize("R,C", [(65, 33), (1, 7), (7, 1), (129, 1153)])
def test_transpose_elementwise_path_exact(R, C):
    """transpose with odd shapes and an odd output row stride (the element-wise path, taken whenever a pair access could be
    misaligned): out (C, R) is a column slice, starting one element in, of a sentinel-filled buffer; the input a column slice of
    a NaN-padded buffer.  A transpose moves bits: out must equal a^T bit for bit and the sentinel must stay."""
    abuf = torch.full((R, C + 5), float("nan"), dtype=torch.bfloat16, device=DEV)
    a = abuf[:, 2:2 + C]
    a.copy_(_randn(R, C, seed=R * 7 + C))
    ldo = R + 2 if (R + 2) % 2 else R + 3
    obuf = torch.full((C, ldo), SENTINEL, dtype=torch.bfloat16, device=DEV)
    out = obuf[:, 1:1 + R]
    before = obuf.clone()
    lib.transpose(a, out)
    assert torch.equal(out.view(torch.int16), a.t().contiguous().view(torch.int16))
    mask = torch.ones_like(obuf, dtype=torch.bool)
    mask[:, 1:1 + R] = False
    assert torch.equal(obuf[mask], before[mask]), "the sentinel around out was written"


# ------------------------------------------------------------------------------------------------- attention backward, BlockFn layouts
@pytest.mark.parametrize("layout", ["packed", "interleaved"])
def test_flash_attn_bwd_one_key_per_query_block_layouts(layout):
    """test_numerics_gpu's one-key backward construction (q_i = 8 k_pi(i), +-1 keys, integer v in +-[1, 4] and dO in [-4, 4]) in the two
    layouts BlockFn uses, with Nq = 201 (a partial 128-row tile and a partial 64-row block):
      packed:      cross-attention, q (B Nq, H 72), keys / values packed rows of a (sum L, 2, H, 72) buffer at kv_off, with
                   kv_len = 65, 1, 0 (a partial key block, a single key, an empty sample);
      interleaved: self-attention on the (B N, 3, H, 72) qkv buffer, gradients into the same layout.
    delta must equal sum_d dO o exactly (integers).  dV[j] is the sum of the dO rows that chose key j (bf16 rounding of an
    integer; where that sum is 0, below Nq 2^-margin 4), |dQ|, |dK| <= scale Nk 2^-margin max|dP - delta| 8 (see
    test_flash_attn_bwd_one_key_per_query); an empty sample has dQ = 0 exactly.  Every gradient element must be written
    (the buffers start as the sentinel) and padding columns keep it."""
    H, D = 16, 72
    C = H * D
    Nq = 201
    lens = [65, 1, 0] if layout == "packed" else [Nq, Nq]
    B, Nk = len(lens), max(lens)
    scale = D ** -0.5
    k, q, pi, margin = _one_key_problem(lens, Nq, H, D, seed=100 + len(layout), alpha=8.0)
    m2 = margin * scale * LOG2E if math.isfinite(margin) else math.inf
    assert m2 > 40, m2
    g = torch.Generator().manual_seed(101)
    # v != 0: then o = v[pi] bit for bit (the other keys add < 2^-30 |v[pi]|), so delta is an integer sum
    v = (torch.randint(1, 5, (B, Nk, H, D), generator=g) * (torch.randint(0, 2, (B, Nk, H, D), generator=g) * 2 - 1)).double()
    do = torch.randint(-4, 5, (B, Nq, H, D), generator=g).double()
    bf = lambda t: t.to(torch.bfloat16).to(DEV)
    if layout == "packed":
        offs = [sum(lens[:b]) for b in range(B)]
        rows = sum(lens)
        kvb, _ = _padded(rows, 2 * C, 64, float("nan"), torch.bfloat16)
        for b, L in enumerate(lens):
            kvb[offs[b]:offs[b] + L].view(L, 2, H, D)[:, 0] = bf(k[b, :L])
            kvb[offs[b]:offs[b] + L].view(L, 2, H, D)[:, 1] = bf(v[b, :L])
        qv, _ = _padded(B * Nq, C, 64, float("nan"), torch.bfloat16)
        qv.copy_(bf(q.reshape(B * Nq, C)))
        kk, vv = kvb[:, :C], kvb[:, C:2 * C]
        qs, ks = (qv.stride(0), D), (kvb.stride(0), D)
        kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
        kv_off = torch.tensor(offs, dtype=torch.int32, device=DEV)
        dq, dqbuf = _padded(B * Nq, C, 64, SENTINEL, torch.bfloat16)
        dkv, dkvbuf = _padded(rows, 2 * C, 64, SENTINEL, torch.bfloat16)
        dk, dvv = dkv[:, :C], dkv[:, C:2 * C]
        dqs, dks = (dq.stride(0), D), (dkv.stride(0), D)
        bufs = ((dqbuf, C), (dkvbuf, 2 * C))
    else:
        rows = B * Nk
        qkv = torch.empty(B * Nq, 3, H, D, dtype=torch.bfloat16, device=DEV)
        qkv[:, 0] = bf(q.reshape(B * Nq, H, D))
        qkv[:, 1] = bf(k.reshape(B * Nk, H, D))
        qkv[:, 2] = bf(v.reshape(B * Nk, H, D))
        qv, kk, vv = qkv[:, 0], qkv[:, 1], qkv[:, 2]
        qs = ks = (3 * C, D)
        kv_len = kv_off = None
        dqkv = torch.full_like(qkv, SENTINEL)
        dq, dk, dvv = dqkv[:, 0], dqkv[:, 1], dqkv[:, 2]
        dqs = dks = (3 * C, D)
        bufs = ()
    o = torch.empty(B * Nq, C, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(B, H, Nq, dtype=torch.float32, device=DEV)
    lib.flash_attn(qv, kk, vv, o, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=rows, kv_len=kv_len, kv_off=kv_off, q_strides=qs,
                   k_strides=ks, v_strides=ks, scale=scale, lse=lse)
    dod = bf(do.reshape(B * Nq, C))
    before = [b_.clone() for b_, _ in bufs]
    delta = torch.full((B * H * Nq,), float("nan"), dtype=torch.float32, device=DEV)
    lib.flash_attn_bwd(qv, kk, vv, o, dod, lse, dq, dk, dvv, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=rows, kv_len=kv_len, kv_off=kv_off,
                       q_strides=qs, k_strides=ks, v_strides=ks, dq_strides=dqs, dk_strides=dks, dv_strides=dks, scale=scale,
                       delta=delta)
    torch.cuda.synchronize()
    want_delta = (o.double() * dod.double()).view(B, Nq, H, D).sum(-1).permute(0, 2, 1).reshape(-1)
    assert torch.equal(delta.double(), want_delta), "delta"
    want_dv = torch.zeros(B, Nk, H, D, dtype=torch.float64)
    for b, L in enumerate(lens):
        for h in range(H):
            if L:
                want_dv[b, :, h].index_add_(0, pi[b, h], do[b, :, h])
    key_rows = [(b, j, (offs[b] if layout == "packed" else b * Nk) + j) for b, L in enumerate(lens) for j in range(L)]
    idx = torch.tensor([r_ for _, _, r_ in key_rows])
    gdv = dvv.double().cpu()[idx].view(-1, H, D)
    gdk = dk.double().cpu()[idx].view(-1, H, D)
    wdv = torch.stack([want_dv[b, j] for b, j, _ in key_rows])
    nz = wdv != 0
    assert torch.equal(gdv[nz], wdv[nz].to(torch.bfloat16).double()), "dV"
    assert (gdv[~nz].abs() <= Nq * 2.0 ** -m2 * 4).all(), "dV zero sums"
    bound = scale * Nk * 2.0 ** -m2 * (2 * D * 16.0) * 8.0
    gq = dq.double().cpu().view(B, Nq, H, D)
    for b, L in enumerate(lens):
        if L == 0:
            assert (gq[b] == 0).all(), f"dQ of the empty sample {b}"
    e_q, e_k = gq.abs().max().item(), gdk.abs().max().item()
    print(f"flash_attn_bwd one-key {layout}: margin {m2:.1f} log2 units, max |dQ| {e_q:.2e}, max |dK| {e_k:.2e}, bound {bound:.2e}")
    assert e_q <= max(bound, 1e-30) and e_k <= max(bound, 1e-30)
    for (buf, cols), bb in zip(bufs, before):
        _assert_pad_unchanged(buf, cols, bb, "gradient buffer")
    if layout == "interleaved":
        assert not (dqkv == SENTINEL).any(), "a gradient element was not written"
    else:
        assert not (dq == SENTINEL).any() and not (dkv == SENTINEL).any(), "a gradient element was not written"
