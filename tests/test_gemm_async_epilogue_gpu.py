"""The GEMM epilogue's output tile is reused from tile to tile while the TMA stores of the previous tile may still be reading
it, and the epilogue operand (residual / pre-activation) of the next tile is loaded into it.  A small persistent grid
(max_ctas 1, 2, 3) runs many tiles per CTA through that reuse; every result must be bitwise equal to the same call on the full
grid, with M and N tails, and nothing outside the output may be written."""
import pytest
import torch
import torch.nn.functional as F

from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
DEV = "cuda"
SENTINEL = -7.25


def _randn(*shape, seed=0, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def _padded(M, N, dtype, fill=SENTINEL):
    """An (M, N) view into an (M + 3, N + 24) buffer filled with `fill`: rows and columns outside the view are sentinels."""
    buf = torch.full((M + 3, N + 24), fill, dtype=dtype, device=DEV)
    return buf, buf[:M, :N]


B, RPB, N, K = 2, 500, 392, 256        # M = 1000: 8 row tiles (tail of 104); N = 392: column tail at BN 128 and 192
M = B * RPB
FORMS = ["bias", "gelu", "gelu_aux", "mul_dgelu", "ln_bias", "ln_bias_gelu", "res_f32", "res_f32_byproducts", "res_bf16"]


def _run(form, max_ctas, block_n):
    a, w, bias = _randn(M, K, seed=1), _randn(N, K, seed=2, scale=K ** -0.5), _randn(N, seed=3, scale=0.1)
    gate = _randn(B, N, seed=4, dtype=torch.float32)
    bufs = {}
    kw = dict(max_ctas=max_ctas, block_n=block_n)
    if form.startswith("res_f32"):
        xbuf, x = _padded(M, N, torch.float32)
        x.copy_(_randn(M, N, seed=5, dtype=torch.float32))
        bufs["out"] = xbuf
        kw.update(epilogue=lib.EPI_BIAS_RESIDUAL, residual=x, gate=gate, gate_batch_stride=N, rows_per_batch=RPB)
        if form == "res_f32_byproducts":
            abuf, aux = _padded(M, N, torch.bfloat16)
            stats = torch.full((M, lib.LN_STAT_PARTS, 2), SENTINEL, device=DEV)
            bufs["aux"], bufs["stats"] = abuf, stats
            kw.update(out_aux=aux, aux_scale=1 + _randn(B, N, seed=6, dtype=torch.float32) * 0.3, aux_scale_batch_stride=N,
                      row_stats_out=stats)
        lib.gemm(a, w, bias, x, **kw)
        return bufs
    obuf, out = _padded(M, N, torch.bfloat16)
    bufs["out"] = obuf
    if form == "res_bf16":
        out.copy_(_randn(M, N, seed=7))
        abuf, aux = _padded(M, N, torch.bfloat16)
        bufs["aux"] = abuf
        kw.update(epilogue=lib.EPI_BIAS_RESIDUAL, residual=out, gate=gate, gate_batch_stride=N, rows_per_batch=RPB, out_aux=aux,
                  aux_is_branch=True)
    elif form == "gelu":
        kw.update(epilogue=lib.EPI_BIAS_GELU)
    elif form == "gelu_aux":
        abuf, aux = _padded(M, N, torch.bfloat16)
        bufs["aux"] = abuf
        kw.update(epilogue=lib.EPI_BIAS_GELU_AUX, out_aux=aux)
    elif form == "mul_dgelu":
        pbuf, pre = _padded(M, N, torch.bfloat16)
        pre.copy_(_randn(M, N, seed=8))
        bias = None
        kw.update(epilogue=lib.EPI_MUL_DGELU, residual=pre)
    elif form.startswith("ln_"):
        stats = torch.rand(M, lib.LN_STAT_PARTS, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9)) + 0.5
        u, v = _randn(B, N, seed=10, dtype=torch.float32), _randn(B, N, seed=11, dtype=torch.float32)
        bias = None
        kw.update(epilogue=lib.EPI_LN_BIAS_GELU if form == "ln_bias_gelu" else lib.EPI_LN_BIAS, rows_per_batch=RPB,
                  ln_stats=stats, ln_u=u, ln_v=v, ln_uv_batch_stride=N, ln_dim=K, ln_eps=1e-6)
    lib.gemm(a, w, bias, out, **kw)
    return bufs


@pytest.mark.parametrize("block_n", [128, 192])
@pytest.mark.parametrize("form", FORMS)
def test_small_grid_matches_full_grid_bitwise(form, block_n):
    want = _run(form, 0, block_n)
    for name, buf in want.items():
        if name == "stats":
            continue
        assert torch.equal(buf[M:], torch.full_like(buf[M:], SENTINEL)), name      # rows past M untouched
        assert torch.equal(buf[:, N:], torch.full_like(buf[:, N:], SENTINEL)), name  # columns past N untouched
    for max_ctas in (1, 2, 3):
        got = _run(form, max_ctas, block_n)
        for name in want:
            assert torch.equal(got[name], want[name]), f"{name} at max_ctas {max_ctas}"


def test_virtual_width_convolution_small_widths():
    """W = 104 does not tile: the GEMM runs over lines padded to 128 pixels and the stores drop pixels x >= 104."""
    Bc, H, W, Cin, Cout = 2, 6, 104, 64, 192
    x = _randn(Bc, H, W, Cin, seed=20)
    wt = _randn(Cout, Cin, 3, 3, seed=21, scale=(9 * Cin) ** -0.5)
    bias = _randn(Cout, seed=22, scale=0.1)
    res = _randn(Bc, H, W, Cout, seed=23)
    want = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias.float(), padding=1).permute(0, 2, 3, 1) + res.float()
    n = Bc * H * W * Cout
    flat = torch.full((n + 4096,), SENTINEL, dtype=torch.bfloat16, device=DEV)
    out = flat[:n].view(Bc, H, W, Cout)
    lib.conv3x3_nhwc(x, wt.permute(0, 2, 3, 1).contiguous(), bias, out, residual=res)
    assert po.rel_err(out.float(), want) < 4e-3
    assert torch.equal(flat[n:], torch.full_like(flat[n:], SENTINEL))


@pytest.mark.parametrize("k_splits", [1, 3])
@pytest.mark.parametrize("max_ctas", [1, 2, 3])
def test_wgrad_split_k_small_grid(k_splits, max_ctas):
    rows, n_out, k_in = 1536, 392, 264
    dy, x = _randn(rows, n_out, seed=30), _randn(rows, k_in, seed=31)
    buf = torch.full((n_out + 3, k_in + 24), SENTINEL, dtype=torch.float32, device=DEV)
    dw = buf[:n_out, :k_in]
    dw.fill_(0.25)
    lib.gemm_wgrad(dy, x, dw, k_splits=k_splits, max_ctas=max_ctas)
    assert po.rel_err(dw - 0.25, dy.float().t() @ x.float()) < 2e-4
    assert torch.equal(buf[n_out:], torch.full_like(buf[n_out:], SENTINEL))
    assert torch.equal(buf[:, k_in:], torch.full_like(buf[:, k_in:], SENTINEL))
