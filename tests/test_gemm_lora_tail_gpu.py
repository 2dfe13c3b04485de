"""The GEMM's K-tail (pxa_gemm_lora_bf16): out = epilogue(a w^T + tail_a tail_w^T + bias) for every epilogue LoRA training
uses, across tail widths on both sides of the 64-column K-block boundary, M / N tails and every block_n; the output with a
zero tail_w equals pxa_gemm_bf16 bit for bit; every rejection."""
import pytest
import torch
import torch.nn.functional as F

from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
DEV = "cuda"

M, N, K, RPB = 1000, 1184, 200, 333          # M, N and K tails; 3 samples of 333 rows (+ 1)
EPIS = ["bias", "gelu", "gelu_aux", "dgelu", "res_bf16", "res_f32_branch", "res_f32"]
TAILS = [8, 16, 48, 64, 72, 200]


def _randn(*shape, seed=0, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def _ints(*shape, seed=0, lo=-8, hi=8, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi, shape, generator=g).to(dtype).to(DEV)


def _call(epi, a, w, bias, ta, tw, seed=9, **kw):
    """Run epilogue `epi` (tail when ta is given); returns (out, aux) as fp64 on the host."""
    B = (M + RPB - 1) // RPB
    gate = _randn(B, N, seed=seed, dtype=torch.float32)
    tail = {} if ta is None else dict(tail_a=ta, tail_w=tw)
    bf = dict(dtype=torch.bfloat16, device=DEV)
    out_bf, aux = torch.empty(M, N, **bf), torch.empty(M, N, **bf)
    if epi == "bias":
        lib.gemm(a, w, bias, out_bf, epilogue=lib.EPI_BIAS, **tail, **kw)
        return out_bf, None
    if epi == "gelu":
        lib.gemm(a, w, bias, out_bf, epilogue=lib.EPI_BIAS_GELU, **tail, **kw)
        return out_bf, None
    if epi == "gelu_aux":
        lib.gemm(a, w, bias, out_bf, epilogue=lib.EPI_BIAS_GELU_AUX, out_aux=aux, **tail, **kw)
        return out_bf, aux
    if epi == "dgelu":
        pre = _randn(M, N, seed=seed + 1, scale=2.0)
        lib.gemm(a, w, None, out_bf, epilogue=lib.EPI_MUL_DGELU, residual=pre, **tail, **kw)
        return out_bf, pre
    g = dict(gate=gate, gate_batch_stride=N, rows_per_batch=RPB)
    if epi == "res_bf16":
        res = _randn(M, N, seed=seed + 2)
        lib.gemm(a, w, bias, out_bf, epilogue=lib.EPI_BIAS_RESIDUAL, residual=res, **g, **tail, **kw)
        return out_bf, res
    res = _randn(M, N, seed=seed + 3, dtype=torch.float32)
    out = torch.empty(M, N, dtype=torch.float32, device=DEV)
    if epi == "res_f32_branch":
        lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=res, out_aux=aux, aux_is_branch=True, **g, **tail, **kw)
        return out, aux
    lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=res, rows_per_batch=RPB, **tail, **kw)
    return out, res


def _want(epi, acc, bias, side):
    """fp64 epilogue of acc (+ bias) -> (out, aux) references."""
    B = (M + RPB - 1) // RPB
    gate = _randn(B, N, seed=9, dtype=torch.float32).double().repeat_interleave(RPB, 0)[:M]
    yb = acc + (bias.double() if bias is not None else 0)
    gelu = lambda v: F.gelu(v, approximate="tanh")
    if epi == "bias":
        return yb, None
    if epi in ("gelu", "gelu_aux"):
        return gelu(yb), (yb if epi == "gelu_aux" else None)
    if epi == "dgelu":
        p = side.double().requires_grad_()
        (d,) = torch.autograd.grad(gelu(p).sum(), p)
        return acc * d, None
    if epi == "res_bf16":
        return side.double() + gate * yb, None
    if epi == "res_f32_branch":                  # side is the aux output here; the residual is regenerated from its seed
        return _randn(M, N, seed=12, dtype=torch.float32).double() + gate * yb, yb
    return side.double() + yb, None


@pytest.mark.parametrize("bn", [0, 128, 192, 256])
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("T", TAILS)
def test_tail_against_fp64(T, epi, bn):
    """The tail against fp64 on the same bf16 operands, with the bounds of the existing GEMM tests (bf16 out 4e-3, fp32
    residual out 2e-4, bf16 aux 4e-3)."""
    a, w = _randn(M, K, seed=1), _randn(N, K, seed=2, scale=K ** -0.5)
    ta, tw = _randn(M, T, seed=3), _randn(N, T, seed=4, scale=T ** -0.5)
    bias = None if epi == "dgelu" else _randn(N, seed=5, scale=0.1)
    out, side = _call(epi, a, w, bias, ta, tw, block_n=bn)
    acc = a.double() @ w.double().T + ta.double() @ tw.double().T
    want, want_aux = _want(epi, acc, bias, side)
    tol = 2e-4 if out.dtype == torch.float32 else 4e-3
    assert po.rel_err(out.double(), want) < tol
    if want_aux is not None:
        assert po.rel_err(side.double(), want_aux) < 4e-3


@pytest.mark.parametrize("bn", [0, 128, 192, 256])
@pytest.mark.parametrize("epi", EPIS)
def test_tail_exact_on_integers(epi, bn):
    """Small integer operands make every fp32 sum exact whatever its order: the tail GEMM equals pxa_gemm_bf16 on the
    operands concatenated along K, bit for bit, for T = 72 (one full and one partial tail K-block)."""
    T = 72
    a, w = _ints(M, K, seed=1), _ints(N, K, seed=2, lo=-2, hi=3)
    ta, tw = _ints(M, T, seed=3), _ints(N, T, seed=4, lo=-2, hi=3)
    bias = None if epi == "dgelu" else _ints(N, seed=5)
    got, got_aux = _call(epi, a, w, bias, ta, tw, block_n=bn)
    want, want_aux = _call(epi, torch.cat([a, ta], 1), torch.cat([w, tw], 1), bias, None, None, block_n=bn)
    assert torch.equal(got, want)
    if got_aux is not None:
        assert torch.equal(got_aux, want_aux)


@pytest.mark.parametrize("bn", [0, 128, 192, 256])
@pytest.mark.parametrize("epi", EPIS)
def test_zero_tail_is_bitwise_the_plain_gemm(epi, bn):
    a, w = _randn(M, K, seed=1), _randn(N, K, seed=2, scale=K ** -0.5)
    bias = None if epi == "dgelu" else _randn(N, seed=5, scale=0.1)
    ta, tw = _randn(M, 16, seed=3), torch.zeros(N, 16, dtype=torch.bfloat16, device=DEV)
    got, got_aux = _call(epi, a, w, bias, ta, tw, block_n=bn)
    want, want_aux = _call(epi, a, w, bias, None, None, block_n=bn)
    assert torch.equal(got, want)
    if got_aux is not None:
        assert torch.equal(got_aux, want_aux)


def test_tail_rejections():
    a, w = _randn(256, 128, seed=1), _randn(256, 128, seed=2)
    out = torch.empty(256, 256, dtype=torch.bfloat16, device=DEV)
    ta, tw = _randn(256, 16, seed=3), _randn(256, 16, seed=4)

    def rejects(code, **kw):
        with pytest.raises(lib.PxaError, match=rf"\({code}\)"):
            lib.gemm(a, w, None, out, **{"tail_a": ta, "tail_w": tw, **kw})

    rejects(-1, epilogue=lib.EPI_LN_BIAS)
    rejects(-1, epilogue=lib.EPI_LN_BIAS_GELU)
    rejects(-1, tail_a=_randn(256, 12, seed=3), tail_w=_randn(256, 12, seed=4))             # tail_k % 8
    buf = torch.zeros(256 * 24 + 8, dtype=torch.bfloat16, device=DEV)
    rejects(-2, tail_a=buf[4:4 + 256 * 24].view(256, 24)[:, :16])                              # misaligned pointer
    rejects(-2, tail_a=buf[:256 * 20].view(256, 20)[:, :16])                                   # stride not a multiple of 8
    rejects(-2, tail_w=buf[:256 * 20].view(256, 20)[:, :16])
    # operands_mn_major (the weight-gradient form) takes no tail
    args = lib.GemmArgs(a=a.data_ptr(), w=w.data_ptr(), out=out.data_ptr(), residual=out.data_ptr(), rows_per_batch=256,
                        M=256, N=256, K=128, lda=256, ldw=256, ldo=256, epilogue=lib.EPI_BIAS_RESIDUAL,
                        out_dtype=lib.DTYPE_F32, operands_mn_major=1)
    tail = lib.GemmTail(tail_a=ta.data_ptr(), tail_w=tw.data_ptr(), tail_k=16, lda_tail=16, ldw_tail=16)
    import ctypes
    assert lib.load().pxa_gemm_lora_bf16(ctypes.byref(args), ctypes.byref(tail), None) == -1
    assert lib.load().pxa_gemm_lora_bf16(ctypes.byref(args), None, None) == -1
