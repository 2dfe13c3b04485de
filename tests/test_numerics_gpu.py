"""Element-wise numerics of the sm_90a kernels (-m gpu) against float64 references computed from the same bf16 inputs.

The normwise `rel_err < tol` checks of the other GPU files miss three kinds of defect: a few wrong elements in a large output
(a tail tile, a padding column), errors where the value is small (normwise error is carried by the large elements), and
statistics that cancel on inputs with a large mean.  The tests here close those gaps:

- Exact constructions: inputs for which the correct output is representable and the kernel's arithmetic on it is exact
  (selection-matrix GEMMs, one-tap convolutions, attention where each query picks one key).  They demand `torch.equal`, so a
  single wrong element fails; each docstring says why exactness holds.
- Guard bands: outputs are written into row-strided slices of wider buffers filled with a sentinel, which must come back
  bit-unchanged, and inputs are read through slices whose padding is NaN, which must not reach the result.
- Element-wise ulp contracts (`assert_bf16_close`) for the transcendental epilogues and the normalisations, over every finite
  bf16 input for the GELU and at |mean| / std up to 128 for the norms; each bound states where its slack comes from.

The helpers print the measured figures (max ulp error, fraction correctly rounded, mean signed ulp error) with `-s`.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from norm_bounds import ln_slack as _ln_slack

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
DEV = "cuda"
K0, K1 = 0.7978845608028654, 0.044715
TINY = 2.0 ** -40
LOG2E = 1.4426950408889634


# ------------------------------------------------------------------------------------------------- shared reference helpers
def bf16_ulp(ref: torch.Tensor) -> torch.Tensor:
    """The spacing of bf16 numbers at |ref| (float64): 2^(e - 7) for |ref| in [2^e, 2^(e+1)), 2^-133 in the subnormal range."""
    _, e = torch.frexp(ref.abs())
    return torch.ldexp(torch.ones_like(ref), (e - 8).clamp(min=-133))


def assert_bf16_close(got: torch.Tensor, ref: torch.Tensor, slack=None, *, name: str, max_ulp: float = 1.0,
                      tiny: float = 0.0, max_bias: float = 0.1) -> None:
    """Element-wise: |got - ref| <= max_ulp * ulp(ref) + slack wherever |ref| > tiny, and |got| <= tiny + slack elsewhere;
    non-finite references must be matched exactly (NaN where NaN, the same infinity).  Also asserts that the mean signed error,
    in ulps, is below max_bias: correct rounding is unbiased, truncation or a biased formula is not, yet stays far under any
    normwise bound.  `slack`: an optional element-wise absolute allowance (e.g. for fp32 accumulation), stated by the caller."""
    got, ref = got.double(), ref.double()
    slack = torch.zeros_like(ref) if slack is None else torch.as_tensor(slack, dtype=torch.float64, device=ref.device).expand_as(ref)
    got, ref, slack = got.flatten(), ref.flatten(), slack.flatten()
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isnan(got[~fin]), torch.isnan(ref[~fin])), f"{name}: NaN pattern differs"
    nn_ = ~fin & ~torch.isnan(ref)
    assert torch.equal(got[nn_], ref[nn_]), f"{name}: infinities differ"
    got, ref, slack = got[fin], ref[fin], slack[fin]
    assert torch.isfinite(got).all(), f"{name}: {(~torch.isfinite(got)).sum().item()} non-finite results for finite references"
    big = ref.abs() > tiny
    ulp = bf16_ulp(ref)
    diff = got - ref
    err_ulp = (diff.abs() / ulp)[big]
    bad = torch.where(big, diff.abs() > max_ulp * ulp + slack, got.abs() > tiny + slack)
    rounded = (got == ref.to(torch.bfloat16).double()).double().mean().item()
    bias = (diff / ulp)[big].mean().item() if big.any() else 0.0
    worst = err_ulp.max().item() if big.any() else 0.0
    print(f"{name}: {ref.numel()} elements, max {worst:.3f} ulp, correctly rounded {rounded:.5f}, mean signed error "
          f"{bias:+.4f} ulp, outside the bound {bad.sum().item()}")
    if bad.any():
        i = torch.nonzero(bad)[:5, 0]
        raise AssertionError(f"{name}: {bad.sum().item()} elements outside the bound, e.g. got {got[i].tolist()} want "
                             f"{ref[i].tolist()}")
    assert abs(bias) <= max_bias, f"{name}: mean signed error {bias:+.4f} ulp"


def gelu64(x: torch.Tensor):
    """float64 GELU(tanh), its derivative and the sum of the derivative's two term magnitudes.  Written as x * sigmoid(2u),
    which equals 0.5 x (1 + tanh u) exactly but does not lose float64's accuracy to the cancellation of 1 + tanh u below
    x = -6 (test_numerics_cpu checks the two agree where float64 evaluates both accurately)."""
    x = x.double()
    u = K0 * (x + K1 * x ** 3)
    du = K0 * (1 + 3 * K1 * x * x)
    e = torch.exp(-2 * u)
    s = 1 / (1 + e)
    t2 = s * (2 * x * (1 / (1 + 1 / e)) * du)             # s * 2 x (1 - s) u', 1 - s = e / (1 + e) also where e overflows
    return x * s, s + t2, s.abs() + t2.abs()


def all_finite_bf16() -> torch.Tensor:
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    return v[torch.isfinite(v.float())].to(DEV)


def _ints(*shape, lo, hi, seed, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g).to(dtype).to(DEV)


def _randn(*shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def _padded(rows, cols, pad, fill, dtype):
    """A (rows, cols) view with row stride cols + pad into a buffer filled with `fill`; returns (view, buffer)."""
    buf = torch.full((rows, cols + pad), fill, dtype=dtype, device=DEV)
    return buf[:, :cols], buf


def _assert_pad_unchanged(buf, cols, before, name):
    assert torch.equal(buf[:, cols:], before[:, cols:]), f"{name}: the padding past column {cols} was written"


SENTINEL = -1280.0        # exactly representable in bf16 (5 x 2^8) and fp32


# ------------------------------------------------------------------------------------------------- D. GELU over every bf16 value
def test_gelu_elementwise_kernel_every_bf16_value():
    """lib.gelu_tanh forward, and backward with dh = 1, over every finite bf16 value plus +-inf.  Contract: <= 1 ulp of the
    float64 value where |ref| > 2^-40, |got| <= 2^-40 elsewhere; the derivative gets 2^-20 (|s| + |2 x s (1-s) u'|) of slack
    (fp32 rounding of its two terms, test_numerics_cpu shows the bound is attainable).  +-inf map as torch maps them."""
    x = all_finite_bf16()
    inf = torch.tensor([float("inf"), float("-inf")], dtype=torch.bfloat16, device=DEV)
    n = x.numel() + 2
    pre = torch.zeros(((n + 1023) // 1024) * 1024, dtype=torch.bfloat16, device=DEV)
    pre[:x.numel()] = x
    pre[x.numel():n] = inf
    ref, dref, dterms = gelu64(x)
    out = lib.gelu_tanh(pre)
    dout = lib.gelu_tanh(pre, dh=torch.ones_like(pre))
    torch.cuda.synchronize()
    assert_bf16_close(out[:x.numel()], ref, name="gelu_tanh forward", tiny=TINY)
    assert_bf16_close(dout[:x.numel()], dref, 2.0 ** -20 * dterms, name="gelu_tanh backward (dh = 1)", tiny=TINY)
    ti = inf.float().requires_grad_(True)
    tf = F.gelu(ti, approximate="tanh")
    tf.sum().backward()
    assert torch.equal(out[x.numel():n].float().isnan(), tf.detach().isnan())
    assert torch.equal(out[x.numel():n].float().nan_to_num(0.0), tf.detach().nan_to_num(0.0))
    assert torch.equal(dout[x.numel():n].float().isnan(), ti.grad.isnan())


def _sweep_matrix():
    """Every finite bf16 value laid out in a (256, 256) bf16 matrix (zero padded), and the 256 x 256 identity: a GEMM
    a @ I^T routes each value unchanged into the fp32 accumulator (one product by 1, the rest by 0 -- exact)."""
    x = all_finite_bf16()
    a = torch.zeros(256 * 256, dtype=torch.bfloat16, device=DEV)
    a[:x.numel()] = x
    return a.view(256, 256), torch.eye(256, dtype=torch.bfloat16, device=DEV)


def test_gemm_gelu_epilogues_every_bf16_value():
    """EPI_BIAS_GELU and EPI_BIAS_GELU_AUX with every finite bf16 value as the pre-activation (routed into the accumulator by
    an identity weight, so the epilogue sees the exact value): out within the GELU contract above, aux == the input bit for
    bit (it is acc + 0 stored to bf16)."""
    a, eye = _sweep_matrix()
    ref = gelu64(a.flatten())[0]
    out = torch.empty_like(a)
    lib.gemm(a, eye, None, out, epilogue=lib.EPI_BIAS_GELU)
    assert_bf16_close(out, ref, name="EPI_BIAS_GELU", tiny=TINY)
    out2, aux = torch.empty_like(a), torch.empty_like(a)
    lib.gemm(a, eye, None, out2, epilogue=lib.EPI_BIAS_GELU_AUX, out_aux=aux)
    assert_bf16_close(out2, ref, name="EPI_BIAS_GELU_AUX", tiny=TINY)
    assert torch.equal(aux.float(), a.float())


def test_gemm_dgelu_epilogue_every_bf16_value():
    """EPI_MUL_DGELU: out = acc * gelu'(pre) with acc = 1 (ones @ I^T, exact) and pre = every finite bf16 value (passed as the
    residual), so out is gelu'(pre) itself: the derivative contract (1 ulp + 2^-20 of its two terms)."""
    pre, eye = _sweep_matrix()
    ones = torch.ones_like(pre)
    out = torch.empty_like(pre)
    lib.gemm(ones, eye, None, out, epilogue=lib.EPI_MUL_DGELU, residual=pre)
    _, dref, dterms = gelu64(pre.flatten())
    assert_bf16_close(out, dref, 2.0 ** -20 * dterms, name="EPI_MUL_DGELU", tiny=TINY)


# ------------------------------------------------------------------------------------------------- B/C. GEMM: exact epilogues
def _selection(N, K):
    """w[n, sigma(n)] = 1, else 0, with sigma(n) = (7 n + 3) mod K: for N >= K every input column is selected (7 is prime to
    the K used here), including the K tail 192..199 of K = 200."""
    sig = (torch.arange(N, device=DEV) * 7 + 3) % K
    w = torch.zeros(N, K, dtype=torch.bfloat16, device=DEV)
    w[torch.arange(N, device=DEV), sig] = 1
    return w, sig


GEMM_EPIS = ["bias", "gelu", "gelu_aux", "dgelu", "res_f32_aux", "res_f32_branch", "res_f32_inplace", "res_bf16", "res_f32_rpb96"]


@pytest.mark.parametrize("bn,max_ctas,reverse", [(0, 0, False), (128, 0, False), (192, 3, False), (256, 0, True), (192, 0, True)])
@pytest.mark.parametrize("epi", GEMM_EPIS)
def test_gemm_selection_matrix_exact(epi, bn, max_ctas, reverse):
    """M = 1000, N = 1184, K = 200 (M, N and K tails; 1184 columns leave an odd number of 32-column chunks in the last tile).
    w is a selection matrix, so acc[:, n] = a[:, sigma(n)] exactly (one product by 1).  a and bias are small integers, gates
    powers of two, residuals multiples of 1/2: every fp32 sum below is exact and, where the output is bf16, representable,
    so the output is compared with torch.equal -- except the GELU outputs, which get the element-wise GELU contract.
    a and w are read through slices whose padding columns are NaN (a load past K would poison the accumulators); out / aux
    are slices of sentinel-filled buffers whose padding must come back unchanged."""
    M, N, K, rpb = 1000, 1184, 200, 333
    if epi == "res_f32_rpb96":
        rpb = 96
    B = (M + rpb - 1) // rpb
    a, _ = _padded(M, K, 56, float("nan"), torch.bfloat16)
    a.copy_(_ints(M, K, lo=-16, hi=15, seed=1))
    w, _ = _padded(N, K, 40, float("nan"), torch.bfloat16)
    sel, sig = _selection(N, K)
    w.copy_(sel)
    bias = _ints(N, lo=-16, hi=15, seed=2)
    yb = a.double()[:, sig] + bias.double()                       # acc + bias, exact
    kw = dict(block_n=bn, max_ctas=max_ctas, reverse_tiles=reverse)
    g = torch.Generator().manual_seed(3)
    if epi in ("bias", "gelu", "gelu_aux", "dgelu"):
        out, obuf = _padded(M, N, 64, SENTINEL, torch.bfloat16)
        aux, abuf = _padded(M, N, 64, SENTINEL, torch.bfloat16)
        before, abefore = obuf.clone(), abuf.clone()
        if epi == "bias":
            lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS, **kw)
            assert torch.equal(out.double(), yb)
        elif epi == "gelu":
            lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_GELU, **kw)
            assert_bf16_close(out, gelu64(yb)[0], name="EPI_BIAS_GELU selection", tiny=TINY)
        elif epi == "gelu_aux":
            lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_GELU_AUX, out_aux=aux, **kw)
            assert_bf16_close(out, gelu64(yb)[0], name="EPI_BIAS_GELU_AUX selection", tiny=TINY)
            assert torch.equal(aux.double(), yb)
            _assert_pad_unchanged(abuf, N, abefore, "out_aux")
        else:
            pre = aux
            pre.copy_(_randn(M, N, seed=4, scale=3.0))
            abefore = abuf.clone()
            lib.gemm(a, w, None, out, epilogue=lib.EPI_MUL_DGELU, residual=pre, **kw)
            acc = a.double()[:, sig]
            _, d, dt = gelu64(pre)
            # acc * gelu'(pre): the product by an exact integer acc adds one fp32 rounding, covered by the 2^-20 slack
            assert_bf16_close(out, acc * d, 2.0 ** -20 * acc.abs() * dt, name="EPI_MUL_DGELU selection", tiny=TINY)
            _assert_pad_unchanged(abuf, N, abefore, "pre (residual)")
        _assert_pad_unchanged(obuf, N, before, "out")
        return
    pick = torch.tensor([0.25, 0.5, 1.0, 2.0, -1.0, 4.0])
    if epi == "res_bf16":
        pick = torch.tensor([0.5, 1.0, 2.0, -1.0])
    gate = pick[torch.randint(0, len(pick), (B, N), generator=g)].to(DEV)
    gate_rows = gate.double().repeat_interleave(rpb, 0)[:M]
    kw.update(gate=gate, gate_batch_stride=N, rows_per_batch=rpb)
    if epi == "res_bf16":
        out, obuf = _padded(M, N, 64, SENTINEL, torch.bfloat16)
        res, _ = _padded(M, N, 64, SENTINEL, torch.bfloat16)
        res.copy_(_ints(M, N, lo=-32, hi=32, seed=5))
        before = obuf.clone()
        want = res.double() + gate_rows * yb                      # |want| <= 96 in steps of 1/2: a bf16 value
        lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=res, **kw)
        assert torch.equal(out.double(), want)
        _assert_pad_unchanged(obuf, N, before, "out")
        return
    out, obuf = _padded(M, N, 64, SENTINEL, torch.float32)
    res0 = _ints(M, N, lo=-128, hi=128, seed=6, dtype=torch.float32) * 0.5
    want = res0.double() + gate_rows * yb                         # fp32-exact: halves plus quarter-multiples, |.| < 2^10
    if epi == "res_f32_inplace":
        out.copy_(res0)
        before = obuf.clone()
        lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=out, **kw)
        assert torch.equal(out.double(), want)
        _assert_pad_unchanged(obuf, N, before, "out")
        return
    res, _ = _padded(M, N, 64, SENTINEL, torch.float32)
    res.copy_(res0)
    aux, abuf = _padded(M, N, 64, SENTINEL, torch.bfloat16)
    before, abefore = obuf.clone(), abuf.clone()
    branch = epi == "res_f32_branch"
    lib.gemm(a, w, bias, out, epilogue=lib.EPI_BIAS_RESIDUAL, residual=res, out_aux=aux, aux_is_branch=branch, **kw)
    assert torch.equal(out.double(), want)
    # aux: the correctly rounded bf16 of an exact fp32 value (the epilogue rounds once, to nearest even)
    assert torch.equal(aux, (yb if branch else want).float().to(torch.bfloat16))
    _assert_pad_unchanged(obuf, N, before, "out")
    _assert_pad_unchanged(abuf, N, abefore, "out_aux")


@pytest.mark.parametrize("k_splits", [0, 1, 2, 3, 4, 5])
def test_gemm_wgrad_one_hot_rows_exact(k_splits):
    """Weight gradient dW += dY^T X with each row r of dY one-hot at column pi(r) = (5 r + 1) mod 200: dW[m] gains the sum
    of the X rows that chose m.  X and the initial dW are small integers, so every partial sum of every K split is an
    integer below 2^24 and exact in fp32 whatever the order of the reduce-adds: torch.equal.  dW is a slice of a
    sentinel-filled buffer."""
    rows, M, N = 1000, 200, 1184
    pi = (torch.arange(rows, device=DEV) * 5 + 1) % M
    dy = torch.zeros(rows, M, dtype=torch.bfloat16, device=DEV)
    dy[torch.arange(rows, device=DEV), pi] = 1
    x = _ints(rows, N, lo=-8, hi=8, seed=7)
    out, obuf = _padded(M, N, 64, SENTINEL, torch.float32)
    out.copy_(_ints(M, N, lo=-100, hi=100, seed=8, dtype=torch.float32))
    want = out.double() + dy.double().T @ x.double()
    before = obuf.clone()
    lib.gemm_wgrad(dy, x, out, k_splits=k_splits)
    assert torch.equal(out.double(), want)
    _assert_pad_unchanged(obuf, N, before, "dW")


# ------------------------------------------------------------------------------------------------- conv3x3: one tap per channel
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 32, 32, 128, 128), (2, 8, 128, 64, 256), (1, 4, 256, 128, 128),
                                            (1, 16, 16, 512, 512), (1, 64, 64, 256, 128),
                                            (1, 24, 104, 64, 128), (1, 16, 152, 128, 128), (2, 5, 24, 64, 64), (1, 12, 208, 64, 256),
                                            (1, 5, 32, 64, 128), (2, 3, 300, 64, 72), (1, 7, 129, 128, 192)])
@pytest.mark.parametrize("with_res", [False, True])
def test_conv3x3_one_tap_exact(B, H, W, Cin, Cout, with_res):
    """Output channel o has one weight of 1, at tap (o mod 9) and input channel (5 o + 1) mod Cin: out[.., o] is the input
    channel shifted by the tap, zero past the border (the kernel's TMA zero fill, and for W = 104, 129, 152, 208, 300 the
    virtual width).  Inputs are small integers, residuals too, so every sum is exact: torch.equal (the output buffer starts
    as NaN, so an unwritten pixel fails as well)."""
    x = _ints(B, H, W, Cin, lo=-16, hi=15, seed=9)
    o = torch.arange(Cout, device=DEV)
    w = torch.zeros(Cout, 3, 3, Cin, dtype=torch.bfloat16, device=DEV)
    w[o, (o % 9) // 3, o % 3, (5 * o + 1) % Cin] = 1
    res = _ints(B, H, W, Cout, lo=-64, hi=64, seed=10) if with_res else None
    out = torch.full((B, H, W, Cout), float("nan"), dtype=torch.bfloat16, device=DEV)
    lib.conv3x3_nhwc(x, w, None, out, residual=res)
    want = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1)
    if with_res:
        want = want + res.double()
    assert torch.equal(out.double(), want)


# ------------------------------------------------------------------------------------------------- attention: one key per query
def _one_key_problem(lens, Nq, H, D, seed, alpha):
    """Keys with +-1 entries (bf16-exact), per (sample, head) a map pi from queries onto every valid key, q_i = alpha k_pi(i).
    Returns k (B, Nk, H, D), q (B, Nq, H, D), pi (B, H, Nq) and the smallest margin, in log2 units of the softmax, by which the
    chosen key's logit beats every other valid key (scale D^-0.5 for d72, 1 for T5)."""
    B, Nk = len(lens), max(max(lens), 1)
    g = torch.Generator().manual_seed(seed)
    k = (torch.randint(0, 2, (B, Nk, H, D), generator=g) * 2 - 1).double()
    pi = torch.zeros(B, H, Nq, dtype=torch.long)
    q = torch.zeros(B, Nq, H, D, dtype=torch.float64)
    margin = math.inf
    for b, L in enumerate(lens):
        if L == 0:
            continue
        for h in range(H):
            perm = torch.randperm(L, generator=g)
            p = perm[torch.arange(Nq) % L]
            pi[b, h] = p
            q[b, :, h] = alpha * k[b, p, h]
            s = q[b, :, h] @ k[b, :L, h].T
            own = s.gather(1, p[:, None])
            s.scatter_(1, p[:, None], -math.inf)
            margin = min(margin, (own[:, 0] - s.max(1).values).min().item())
    return k, q, pi, margin


@pytest.mark.parametrize("layout", ["padded", "packed", "interleaved"])
@pytest.mark.parametrize("fp32_p", [False, True])
def test_flash_attn_one_key_per_query_exact(layout, fp32_p):
    """q_i = 8 k_pi(i) with +-1 keys: the chosen logit beats every other valid key by more than 8 in log2 units (asserted),
    so when its key block arrives the running max becomes that logit (the forward takes the max and rescales O by corr in
    every block) and its P is exp2(0) = 1 exactly; every other P is < 2^-margin.  The normaliser is then 1 + (< 2^-20), and with
    1/2 <= |v| < 3/2 the other keys add < 2^-30 |v[pi(i)]|, far below half a bf16 ulp, so out[i] == v[pi(i)] bit for bit (a v
    element of 0 would instead receive those tiny terms, correctly, and is therefore excluded), and lse[i] = logit * log2 e to fp32 accuracy.  pi maps onto every valid
    key (keys 63 / 64 / 127 / 128 and the partial last block included); ragged kv_len with an empty sample (zero output), 16
    heads with their own pi, packed kv_off, the interleaved qkv buffer.  q / k / v are read with a head stride of 80 whose 8
    padding columns are NaN (the 64 + 64 column split of head_dim 72 must zero-fill columns 72..127, not load them), and out
    is a slice of a sentinel-filled buffer (ldo > H * 72)."""
    H, D, Nk = 16, 72, 256
    lens = [256, 129, 0, 200] if layout != "interleaved" else [256, 256]
    Nq = Nk if layout == "interleaved" else 320
    B = len(lens)
    scale = D ** -0.5
    k, q, pi, margin = _one_key_problem(lens, Nq, H, D, seed=11, alpha=8.0)
    assert margin * scale * LOG2E > 20, margin
    g = torch.Generator().manual_seed(12)
    v = ((torch.rand(B, Nk, H, D, generator=g) + 0.5) * (torch.randint(0, 2, (B, Nk, H, D), generator=g) * 2 - 1))
    v = v.to(torch.bfloat16).double()
    HS = 80
    if layout == "interleaved":                 # (B*N, 3, H, 80): q / k / v of one token side by side, as the QKV GEMM writes
        buf = torch.full((B * Nk, 3, H, HS), float("nan"), dtype=torch.bfloat16, device=DEV)
        buf[:, 0, :, :D] = q.reshape(B * Nq, H, D).to(torch.bfloat16).to(DEV)
        buf[:, 1, :, :D] = k.reshape(B * Nk, H, D).to(torch.bfloat16).to(DEV)
        buf[:, 2, :, :D] = v.reshape(B * Nk, H, D).to(torch.bfloat16).to(DEV)
        qv, kv_, vv = buf[:, 0], buf[:, 1], buf[:, 2]
        qs = ks = vs = (3 * H * HS, HS)
        kv_len, kv_off, kv_rows = None, None, B * Nk
    else:
        qb = torch.full((B * Nq, H, HS), float("nan"), dtype=torch.bfloat16, device=DEV)
        qb[:, :, :D] = q.reshape(B * Nq, H, D).to(torch.bfloat16).to(DEV)
        qv, qs = qb, (H * HS, HS)
        if layout == "padded":
            kb = torch.full((B * Nk, 2, H, HS), float("nan"), dtype=torch.bfloat16, device=DEV)
            kb[:, 0, :, :D] = k.reshape(B * Nk, H, D).to(torch.bfloat16).to(DEV)
            kb[:, 1, :, :D] = v.reshape(B * Nk, H, D).to(torch.bfloat16).to(DEV)
            kv_off, kv_rows = None, B * Nk
        else:                                   # packed: sample b's keys start at row off[b], no rows between samples
            offs = [sum(lens[:b]) for b in range(B)]
            kv_rows = sum(lens)
            kb = torch.full((kv_rows, 2, H, HS), float("nan"), dtype=torch.bfloat16, device=DEV)
            for b, L in enumerate(lens):
                kb[offs[b]:offs[b] + L, 0, :, :D] = k[b, :L].to(torch.bfloat16).to(DEV)
                kb[offs[b]:offs[b] + L, 1, :, :D] = v[b, :L].to(torch.bfloat16).to(DEV)
            kv_off = torch.tensor(offs, dtype=torch.int32, device=DEV)
        kv_, vv = kb[:, 0], kb[:, 1]
        ks = vs = (2 * H * HS, HS)
        kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    out, obuf = _padded(B * Nq, H * D, 64, SENTINEL, torch.bfloat16)
    before = obuf.clone()
    lse = torch.full((B, H, Nq), float("nan"), dtype=torch.float32, device=DEV)
    lib.flash_attn(qv, kv_, vv, out, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=kv_rows, kv_len=kv_len, kv_off=kv_off, q_strides=qs,
                   k_strides=ks, v_strides=vs, lse=lse, fp32_p=fp32_p)
    torch.cuda.synchronize()
    want = torch.zeros(B, Nq, H, D, dtype=torch.float64)
    want_lse = torch.zeros(B, H, Nq, dtype=torch.float64)
    for b, L in enumerate(lens):
        if L == 0:
            continue
        for h in range(H):
            want[b, :, h] = v[b, pi[b, h], h]
            want_lse[b, h] = (q[b, :, h] * k[b, pi[b, h], h]).sum(-1) * scale * LOG2E
    got = out.double().cpu().view(B, Nq, H, D)
    bad = (got != want).any(-1)
    assert not bad.any(), f"{bad.sum().item()} (query, head) rows differ, first at {torch.nonzero(bad)[0].tolist()}"
    _assert_pad_unchanged(obuf, H * D, before, "attention out")
    valid = torch.tensor([L > 0 for L in lens])
    lerr = ((lse.double().cpu() - want_lse).abs() / want_lse.abs().clamp(min=1))[valid].max().item()
    print(f"flash_attn one-key {layout} fp32_p={fp32_p}: margin {margin * scale * LOG2E:.1f} log2 units, lse max rel err {lerr:.2e}")
    assert lerr < 1e-6                        # fp32 logits of +-8 x +-1 products: exact; log2 of 1 + (< 2^-20) adds < 2e-6 / 100


def test_flash_attn_bwd_one_key_per_query():
    """Backward on the one-key construction with integer v and dO: P is one-hot up to < 2^-margin, so dV[j] is the sum of
    the dO rows whose query chose key j plus < Nq 2^-margin 4 from the others (integers: where the sum is not 0 its bf16
    rounding is compared with torch.equal, where it is 0 dV must stay below that), and dS = P (dP - delta)
    vanishes on the chosen key exactly (o = v[pi], so dP = delta in exact integer arithmetic) and elsewhere is below
    |dP - delta| 2^-margin.  Hence |dQ|, |dK| <= scale * Nk * 2^-margin * max|dP - delta| * max|k or q| (stated in the
    assertion, < 1e-6 here).  Rows of dK / dV at or past kv_len, and the padding columns of the dq / dk / dv buffers, keep
    their sentinel."""
    H, D, Nq, Nk = 4, 72, 384, 256
    lens = [256, 100, 0, 129]
    B = len(lens)
    scale = D ** -0.5
    k, q, pi, margin = _one_key_problem(lens, Nq, H, D, seed=13, alpha=8.0)
    m2 = margin * scale * LOG2E
    assert m2 > 40, m2
    g = torch.Generator().manual_seed(14)
    v = torch.randint(-4, 5, (B, Nk, H, D), generator=g).double()
    do = torch.randint(-4, 5, (B, Nq, H, D), generator=g).double()
    bf = lambda t, rows: t.reshape(rows, H * D).to(torch.bfloat16).to(DEV)
    qd, kd, vd, dod = bf(q, B * Nq), bf(k, B * Nk), bf(v, B * Nk), bf(do, B * Nq)
    kl = torch.tensor(lens, dtype=torch.int32, device=DEV)
    st = (H * D, D)
    o = torch.empty(B * Nq, H * D, dtype=torch.bfloat16, device=DEV)
    lse = torch.empty(B, H, Nq, dtype=torch.float32, device=DEV)
    lib.flash_attn(qd, kd, vd, o, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=B * Nk, kv_len=kl, q_strides=st, k_strides=st, v_strides=st,
                   lse=lse)
    dq, dqb = _padded(B * Nq, H * D, 64, SENTINEL, torch.bfloat16)
    dk, dkb = _padded(B * Nk, H * D, 64, SENTINEL, torch.bfloat16)
    dv, dvb = _padded(B * Nk, H * D, 64, SENTINEL, torch.bfloat16)
    bq, bk, bv = dqb.clone(), dkb.clone(), dvb.clone()
    lib.flash_attn_bwd(qd, kd, vd, o, dod, lse, dq, dk, dv, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=B * Nk, kv_len=kl, q_strides=st,
                       k_strides=st, v_strides=st, dq_strides=(dq.stride(0), D), dk_strides=(dk.stride(0), D),
                       dv_strides=(dv.stride(0), D))
    torch.cuda.synchronize()
    want_dv = torch.zeros(B, Nk, H, D, dtype=torch.float64)
    for b, L in enumerate(lens):
        for h in range(H):
            if L:
                want_dv[b, :, h].index_add_(0, pi[b, h], do[b, :, h])
    gdv, gdk = dv.double().cpu().view(B, Nk, H, D), dk.double().cpu().view(B, Nk, H, D)
    dpmax = 2 * D * 16.0                                          # |dP|, |delta| <= 72 * 4 * 4
    bound = scale * Nk * 2.0 ** -m2 * dpmax * 8.0                 # |k| = 1, |q| = 8
    for b, L in enumerate(lens):
        w_, g_ = want_dv[b, :L], gdv[b, :L]
        nz = w_ != 0             # where the dO rows sum to 0, dV holds the other keys' < 2^-margin share instead
        assert torch.equal(g_[nz], w_[nz].to(torch.bfloat16).double()), f"dV of sample {b}"
        assert (g_[~nz].abs() <= Nq * 2.0 ** -m2 * 4).all(), f"dV zero sums of sample {b}"
        assert (gdv[b, L:] == SENTINEL).all() and (gdk[b, L:] == SENTINEL).all(), f"dK / dV rows >= kv_len of sample {b}"
    valid_k = torch.cat([torch.arange(L) + b * Nk for b, L in enumerate(lens)])
    e_q, e_k = dq.double().abs().max().item(), dk.double().cpu()[valid_k].abs().max().item()
    print(f"flash_attn_bwd one-key: margin {m2:.1f} log2 units, max |dQ| {e_q:.2e}, max |dK| {e_k:.2e}, bound {bound:.2e}")
    assert e_q <= max(bound, 1e-30) and e_k <= max(bound, 1e-30)
    for buf, ref, nm in ((dqb, bq, "dq"), (dkb, bk, "dk"), (dvb, bv, "dv")):
        _assert_pad_unchanged(buf, H * D, ref, nm)


def test_t5_attn_one_key_per_query_exact():
    """T5 encoder attention (head_dim 64, scale 1) on the same construction (alpha = 1, +-1 keys) with a relative-position
    bias in [-2, 2] and a key mask: keys >= len_b carry a key_bias of -1e9.  The chosen logit beats every other unmasked key
    by the asserted margin minus 4 (the bias spread), > 8 in log2 units, so out[i] == v[pi(i)] bit for bit; out is a slice of a
    sentinel-filled buffer."""
    B, H, L, D = 2, 4, 300, 64
    lens = [300, 77]
    k, q, pi, margin = _one_key_problem(lens, L, H, D, seed=15, alpha=1.0)
    assert (margin - 4) * LOG2E > 20, margin
    k_full = torch.randn(B, L, H, D, generator=torch.Generator().manual_seed(16)).sign().double()
    for b, Lb in enumerate(lens):
        k_full[b, :Lb] = k[b, :Lb]
    v = torch.randn(B, L, H, D, generator=torch.Generator().manual_seed(17)).to(torch.bfloat16).double()
    bias = (torch.rand(H, L, L, generator=torch.Generator().manual_seed(18)) * 4 - 2).to(DEV)
    key_bias = torch.zeros(B, L)
    for b, Lb in enumerate(lens):
        key_bias[b, Lb:] = -1e9
    bf = lambda t: t.reshape(B * L, H * D).to(torch.bfloat16).to(DEV)
    out, obuf = _padded(B * L, H * D, 64, SENTINEL, torch.bfloat16)
    before = obuf.clone()
    lib.t5_attn(bf(q), bf(k_full), bf(v), out, bias, key_bias.to(DEV), B=B, H=H, L=L, scale=1.0)
    torch.cuda.synchronize()
    want = torch.zeros(B, L, H, D, dtype=torch.float64)
    for b in range(B):
        for h in range(H):
            want[b, :, h] = v[b, pi[b, h], h]
    got = out.double().cpu().view(B, L, H, D)
    bad = (got != want).any(-1)
    assert not bad.any(), f"{bad.sum().item()} (query, head) rows differ"
    _assert_pad_unchanged(obuf, H * D, before, "t5 out")


# ------------------------------------------------------------------------------------------------- E. statistics at large offsets
def _offset_input(shape, ratio, seed):
    """bf16 values ratio + N(0, 1): |mean| / std = ratio."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) + ratio).to(torch.bfloat16).to(DEV)


@pytest.mark.parametrize("ratio", [0, 4, 32, 128])
@pytest.mark.parametrize("B,H,W,Cc,silu", [(2, 64, 48, 256, True), (1, 1024, 1024, 128, True), (1, 256, 256, 512, False)])
def test_groupnorm_large_offsets_elementwise(B, H, W, Cc, silu, ratio):
    """GroupNorm(32) (+ SiLU) against float64 F.group_norm at |mean| / std = ratio, up to the 1024-px decoder's groups
    (128 channels: 4 M elements per group).  Bound: 2 ulp, plus an absolute slack of 2^-16 |gamma| (1 + |xhat|) for the
    group statistics: fp32 sums of 10^3 .. 10^6 terms (per-thread runs, then shared-memory and global atomics in arbitrary
    order) put an error of a few 2^-24 x sqrt(terms) times the spread of x - K on the mean and the variance, well below
    2^-16 of the standard deviation.  With one-pass sums of x itself the variance cancels at ratio 128."""
    x = _offset_input((B, H, W, Cc), ratio, seed=20 + ratio)
    gamma = (1 + _randn(Cc, seed=21, scale=0.1).float()).to(torch.bfloat16)
    beta = _randn(Cc, seed=22, scale=0.1)
    out = torch.full_like(x, float("nan"))
    lib.groupnorm_silu_nhwc(x, gamma, beta, out, groups=32, eps=1e-6, silu=silu)
    xd = x.double().permute(0, 3, 1, 2)
    xhat = F.group_norm(xd, 32, None, None, 1e-6)
    want = xhat * gamma.double()[:, None, None] + beta.double()[:, None, None]
    if silu:
        want = F.silu(want)
    want = want.permute(0, 2, 3, 1)
    slack = 2.0 ** -16 * gamma.double().abs() * (1 + xhat.permute(0, 2, 3, 1).abs())
    del xd, xhat
    assert_bf16_close(out, want, slack, name=f"groupnorm{'+silu' if silu else ''} {B}x{H}x{W}x{Cc} mean/std={ratio}",
                      max_ulp=2.0)


@pytest.mark.parametrize("ratio", [0, 4, 32, 128])
@pytest.mark.parametrize("xdtype", [torch.float32, torch.bfloat16])
def test_ln_modulate_large_offsets_elementwise(xdtype, ratio):
    """ln_modulate (LayerNorm eps 1e-6, no affine, then * (1 + scale_b) + shift_b) at |mean| / std = ratio against float64:
    2 ulp plus the fp32 slack of _ln_slack.  Two-pass statistics in registers: no cancellation."""
    B, Ntok, Cc = 3, 333, 1152
    x = _offset_input((B * Ntok, Cc), ratio, seed=30 + ratio).to(xdtype)
    mod = _randn(B, 6, Cc, seed=31, dtype=torch.float32) * 0.3
    out = torch.empty(B * Ntok, Cc, dtype=torch.bfloat16, device=DEV)
    lib.ln_modulate(x, mod[:, 3], mod[:, 4], out, mod_batch_stride=6 * Cc, rows_per_batch=Ntok)
    xd = x.double()
    xn = F.layer_norm(xd, (Cc,), eps=1e-6)
    m = 1 + mod[:, 4].double().repeat_interleave(Ntok, 0)
    want = xn * m + mod[:, 3].double().repeat_interleave(Ntok, 0)
    r = (xd.mean(1, keepdim=True).abs() / xd.std(1, keepdim=True))
    assert_bf16_close(out, want, _ln_slack(xd, r, m.abs()) + 2.0 ** -22 * want.abs(), max_ulp=2.0,
                      name=f"ln_modulate x={xdtype} mean/std={ratio}")


@pytest.mark.parametrize("ratio", [0, 4, 32, 128])
def test_layernorm_affine_large_offsets_elementwise(ratio):
    """layernorm_affine_ (qk_norm, eps 1e-5) in place on a column slice, at |mean| / std = ratio: 2 ulp plus _ln_slack."""
    M, Cc = 777, 1152
    qkv = _randn(M, 3 * Cc, seed=40)
    qkv[:, :Cc] = _offset_input((M, Cc), ratio, seed=41 + ratio)
    w, b = (1 + _randn(Cc, seed=42, scale=0.1).float()).to(torch.bfloat16), _randn(Cc, seed=43, scale=0.1)
    xd = qkv[:, :Cc].double()
    want = F.layer_norm(xd, (Cc,), w.double(), b.double(), eps=1e-5)
    rest = qkv[:, Cc:].clone()
    lib.layernorm_affine_(qkv[:, :Cc], w, b, eps=1e-5)
    r = xd.mean(1, keepdim=True).abs() / xd.std(1, keepdim=True)
    assert_bf16_close(qkv[:, :Cc], want, _ln_slack(xd, r, w.double().abs()) + 2.0 ** -22 * want.abs(), max_ulp=2.0,
                      name=f"layernorm_affine mean/std={ratio}")
    assert torch.equal(qkv[:, Cc:], rest)


@pytest.mark.parametrize("ratio", [0, 4, 32, 128])
def test_rmsnorm_large_offsets_elementwise(ratio):
    """rmsnorm (T5LayerNorm) at |mean| / std = ratio: no mean is subtracted, the sum of squares is a sum of positive terms,
    so 2 ulp plus 2^-20 relative (fp32 rounding of a 4608-term sum of squares) holds at any offset."""
    M, Cc = 300, 4096
    x = _offset_input((M, Cc), ratio, seed=50 + ratio).float()
    w = (1 + _randn(Cc, seed=51, scale=0.1).float()).to(torch.bfloat16)
    out = torch.empty(M, Cc, dtype=torch.bfloat16, device=DEV)
    lib.rmsnorm(x, w, out, eps=1e-6)
    xd = x.double()
    want = xd * torch.rsqrt((xd * xd).mean(1, keepdim=True) + 1e-6) * w.double()
    assert_bf16_close(out, want, 2.0 ** -20 * want.abs(), max_ulp=2.0, name=f"rmsnorm mean/std={ratio}")


@pytest.mark.parametrize("ratio", [0, 4, 32, 128])
def test_fused_ln_epilogue_error_grows_with_offset_as_designed(ratio):
    """EPI_LN_BIAS (opt-in fused LayerNorm-modulate): out = rstd (acc - mean u) + v with acc = sum_k bf16(x_k m_k) w_nk.  The
    bf16 rounding of x m is relative to |x| ~ |mean|, not to the normalised value, so the error is pinned by
        |out - ref| <= 1 ulp + 1.1 * 2^-9 rstd sum_k |x_k m_k w_nk| + 2^-14 (1 + (mean / std)^2) |ref - v|
    (the second term: every rounding at its worst; the third: one-pass fp32 row statistics, whose variance carries ~2^-18
    (mean / std)^2 relative error).  The bound grows like 1 + |mean| / std: a design trade-off of the fused form, see
    PXA_EPI_LN_BIAS in include/pixart_sm100.h.  Printed: the largest error / bound ratio."""
    B, rpb, K, N = 2, 256, 1152, 384
    M = B * rpb
    x = _offset_input((M, K), ratio, seed=60 + ratio).float()
    shift = _randn(B, K, seed=61, dtype=torch.float32) * 0.3
    scale = _randn(B, K, seed=62, dtype=torch.float32) * 0.3
    w, bias = _randn(N, K, seed=63, scale=K ** -0.5), _randn(N, seed=64, scale=0.1)
    mult = (1 + scale).contiguous()
    a = torch.empty(M, K, dtype=torch.bfloat16, device=DEV)
    stats = torch.empty(M, lib.LN_STAT_PARTS, 2, device=DEV)
    lib.ln_prepare(x, mult, a, stats, mod_batch_stride=K, rows_per_batch=rpb)
    u, v = mult @ w.float().T, shift @ w.float().T + bias.float()
    out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    lib.gemm(a, w, None, out, epilogue=lib.EPI_LN_BIAS, rows_per_batch=rpb, ln_stats=stats, ln_u=u.contiguous(),
             ln_v=v.contiguous(), ln_uv_batch_stride=N, ln_dim=K, ln_eps=1e-6)
    xd = x.double()
    xn = F.layer_norm(xd, (K,), eps=1e-6)
    md = mult.double().repeat_interleave(rpb, 0)
    want = F.linear(xn * md + shift.double().repeat_interleave(rpb, 0), w.double(), bias.double())
    rstd = 1 / torch.sqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-6)
    r = xd.mean(1, keepdim=True).abs() * rstd
    vb = v.double().repeat_interleave(rpb, 0)
    bound = 1.1 * 2.0 ** -9 * rstd * ((xd * md).abs() @ w.double().abs().T) + 2.0 ** -14 * (1 + r * r) * (want - vb).abs()
    err = (out.double() - want).abs()
    worst = (err / (bf16_ulp(want) + bound)).max().item()
    print(f"EPI_LN_BIAS mean/std={ratio}: max |err| {err.max().item():.3e}, max err / bound {worst:.3f}")
    assert worst <= 1.0
