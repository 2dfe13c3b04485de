"""Float64 references and element-wise error bounds for the wgmma GEMM family (gemm_sm100.cu): every epilogue of
pxa_gemm_bf16, the LoRA K-tail of pxa_gemm_lora_bf16, the split-K weight gradient, the implicit-GEMM 3x3 convolution and the
fused LayerNorm chain (pxa_ln_prepare, aux_scale / row_stats_out, EPI_LN_*).  Shared by test_gemm_numerics_cpu.py, which
checks the bounds against float32 emulations of the kernels, and test_gemm_numerics_gpu.py, which checks the kernels against
them.

Every output o is checked as
    |o_kernel - o_ref| <= c ulp(|o_ref| + slack) + slack,
with ulp in the output's dtype, c = 1/2 for the final rounding (1 for the GELU outputs, the GELU's own contract) and `slack` a
first-order bound on everything before it, in float64.  u = 2^-24 is the fp32 unit roundoff.

Accumulator.  The reference is the exact float64 sum acc = sum_k a_k w_k of the same bf16 operands (the products are exact in
float64, and the sums of a few thousand of them lose nothing next to the bounds).  The kernel's order: 64-wide K-blocks, each
issued as 4 wgmma k16 steps into the fp32 accumulator, zero-filled past K; the LoRA tail's ceil(T / 64) K-blocks follow the
last K-block of A W^T; the convolution's K-block kb is (tap kb / (Cin / 64), 64-channel slice), tap-major, which is the
(Cout, 3, 3, Cin) order of the packed weight.  Step s adds the 16-product group G_s to the running sum P_{s-1} with error
    <= 2^-23 (|P_{s-1}| + sum_{k in G_s} |a_k w_k|),
the truncating-adder allowance attn_bounds.py uses too, and the accumulator's slack is the sum over the steps, computed exactly
in float64 from the prefix sums of the group sums (`accumulate`).  It is an allowance, not a worst case of every truncating
adder: an adder that aligns the 17 terms to the largest exponent and truncates each can lose up to 2^-23 max|term| per lossy
term, so a step with one dominant product and 16 tiny ones can exceed it.  On real data the per-step losses carry both signs
and the sum over steps keeps a wide margin; test_gemm_numerics_cpu.py measures it for that model and for sequential fp32.
The shortcut K 2^-23 sum |a w| is not used: at K = 4608 it is about 6 bf16 ulps of a typical element and would accept a
double rounding.  Split-K: each split sums its own K-blocks [ks nkb / k, (ks + 1) nkb / k) from zero, and the k partials are
reduce-added into `out` in an unknown order, each addition rounding once: k u (|bucket| + sum_ks |partial_ks|).

Epilogues (y = acc + bias, formed in fp32: slack_y = slack_acc + u |y|):
  - EPI_BIAS: y.  EPI_BIAS_GELU: gelu(y), 1 ulp (the kernel's GELU contract: 1 bf16 ulp wherever |gelu| > 2^-40, 2^-40
    absolute below) + (|gelu'(y)| + 0.8 slack_y) slack_y (|gelu''| <= 0.8).  EPI_BIAS_GELU_AUX: the same, and aux = y.
  - EPI_MUL_DGELU: acc gelu'(pre), pre the bf16 operand: |gelu'(pre)| slack_acc + 2^-20 |acc| (|s| + |s t2|) + 2^-40, the
    derivative's contract in test_numerics_gpu.py (it covers the fp32 product too; below pre = -9 the derivative, < 1e-37,
    flushes to zero).
  - fp32 residual: out = fmaf(gate, y, r): |gate| slack_y, and the fma's one rounding is the half fp32 ulp.
  - bf16 residual: the same with u |out| for the fp32 fma, then half a bf16 ulp.
  - aux (out, or y with aux_is_branch): the slack of the value it copies, times |aux_scale| when given, + u |aux| for that
    product, then half a bf16 ulp.  The value it copies is the fp32 one: scaling the bf16-rounded out rounds twice.
  - row_stats_out part t: (sum o, sum o^2) over the tile's columns of the fp32 `out` the kernel wrote.  Each thread sums its
    BN / 16 column pairs (pair sums; two fmaf per pair for the squares), 2 shuffle levels, then the two warpgroups' halves:
    depth BN / 16 + 4 (sums) and BN / 8 + 4 (squares), times u sum |.|.  Parts past the last column tile are exactly 0.
  - pxa_ln_prepare: a = bf16(fp32(x mult)): u |x mult|, then half a bf16 ulp.  Statistics: each lane sums 9 float4 as
    (x + y) + (z + w) in sequence (depth 2 + 9), then a 5-level shuffle tree: 16 u sum |x|; the squares are one fmaf chain
    of 36 per lane + 5 levels: 41 u sum x^2.  Parts 1..7 are 0.
  - EPI_LN_BIAS / _GELU: the kernel's formula x = fmaf(rstd, acc, fmaf(-rstd mu, u_b, v_b)) with mu = S / d and
    rstd = rsqrtf(Q / d - mu^2 + eps) from the fp32 partial sums it is given (S, Q: their float64 sums).  The statistics:
    8 u sum|parts| for each fp32 sum of the 8 parts, u for fp32(1 / d), u for each product, so
        e(mu) = 3u |mu| + 8u sum|S parts| / d,  e(Q/d) = 3u Q / d + 8u sum|Q parts| / d,
        e(var) = e(Q/d) + 2 |mu| e(mu) + u mu^2 + u var (+ u (var + eps) for the eps add),
        rel(rstd) = e(var) / (2 (var + eps)) + 2^-22 (rsqrtf: 2 ulp),
        e(c) = |c| (u + rel(rstd)) + rstd e(mu)                                   c = -rstd mu,
        slack = rstd slack_acc + rel(rstd) rstd |acc| + e(c) |u_b| + u |c u_b + v_b| + u |x|.
    The rstd |acc| and e(c) |u| terms grow like |mu| rstd: this is the fused form's trade-off (see
    test_fused_ln_epilogue_error_grows_with_offset_as_designed for its effect against an unfused LayerNorm).

Bias: `Tally` also reports mean(sign(ref) (got - ref) / bound) over the elements with |ref| > `tiny`.  Round to nearest
leaves it near 0; a store that rounds toward zero pulls every element's error towards -sign(ref) and moves the mean by about
-0.5 ulp / bound while each element stays inside its bound.  MAX_BIAS is set from test_gemm_numerics_cpu.py: see there.
It applies to the bf16 outputs, the only ones a store rounds.  On fp32 outputs the statistic measures the accumulator itself:
on an H100 80GB HBM3 (700 W) the wgmma accumulator pulls towards zero more than model (b) of the CPU test does -- bias down to
-0.096 where out is the bare accumulator (K = 1152; model (b): -0.011), -0.03 .. -0.06 for split-K and the gated residuals --
while its largest error stays at 0.37 of the step allowance.  So fp32 outputs are held by the element-wise bound alone.
"""
import math

import torch

U = 2.0 ** -24
U_ACC = 2.0 ** -23
KB = 64                      # K-block
KSTEP = 16                   # wgmma k16 step
GELU2 = 0.8                  # max |gelu''| (0.798 at 0)
GELU_TINY = 2.0 ** -40       # below it the GELU contract is absolute
DGELU = 2.0 ** -20
RSQRT = 2.0 ** -22
K0, K1 = 0.7978845608028654, 0.044715
LN_STAT_PARTS = 8
MAX_BIAS = 0.1               # |mean(sign(ref) err / bound)|; CPU emulations: models within 0.008, truncating stores <= -0.49
SENTINEL = -7.75             # written around outputs; must come back unchanged (exact in bf16 and fp32)


# ------------------------------------------------------------------------------------------------- shared helpers
def bf16_ulp(ref):
    """The spacing of bf16 numbers at |ref| (float64): 2^(e - 8) for |ref| in [2^(e-1), 2^e), 2^-133 below the normals."""
    _, e = torch.frexp(ref.abs())
    return torch.ldexp(torch.ones_like(ref), (e - 8).clamp(min=-133))


def f32_ulp(ref):
    """The spacing of fp32 numbers at |ref| (float64): 2^(e - 24) for |ref| in [2^(e-1), 2^e), 2^-149 below the normals."""
    _, e = torch.frexp(ref.abs())
    return torch.ldexp(torch.ones_like(ref), (e - 24).clamp(min=-149))


def gelu64(x):
    """float64 GELU(tanh) as x sigmoid(2u), its derivative and the sum of the derivative's two term magnitudes."""
    x = x.double()
    u = K0 * (x + K1 * x ** 3)
    du = K0 * (1 + 3 * K1 * x * x)
    e = torch.exp(-2 * u)
    s = 1 / (1 + e)
    t2 = s * (2 * x * (1 / (1 + 1 / e)) * du)
    return x * s, s + t2, s.abs() + t2.abs()


def nan_padded(t, pad=8, dtype=None):
    """A copy of the 2-D `t` (as `dtype`) in a row-strided buffer whose pad columns are NaN: a kernel that reads past the
    row's end returns NaN."""
    dtype = dtype or t.dtype
    rows, cols = t.shape
    buf = torch.full((rows, cols + pad), float("nan"), dtype=dtype, device=t.device)
    buf[:, :cols] = t
    return buf[:, :cols]


def sentinel_out(M, N, dtype, device, pad=8, fill=None):
    """(view, buffer): an (M, N) row-strided view of an (M + 1, N + pad) buffer filled with SENTINEL; `fill` (M, N), when
    given, is copied into the view (an in-place residual)."""
    buf = torch.full((M + 1, N + pad), SENTINEL, dtype=dtype, device=device)
    view = buf[:M, :N]
    if fill is not None:
        view.copy_(fill)
    return view, buf


def assert_guard(buf, M, N, name):
    """The guard band of a `sentinel_out` buffer (columns past N, the row past M) came back unchanged."""
    band = torch.cat([buf[:M, N:].flatten(), buf[M:].flatten()]).float()
    bad = (band != SENTINEL).sum().item()
    assert bad == 0, f"{name}: {bad} guard elements overwritten"


def auto_splits(M, N, K, sms):
    """The split count launch_wgrad picks for k_splits = 0 (gemm_sm100.cu) on `sms` SMs: the most even wave."""
    tiles = -(-M // 128) * -(-N // 128)
    nkb = -(-K // 64)
    best, best_eff, ks = 1, 0.0, 1
    while ks <= 16 and nkb // ks >= 8:
        t = tiles * ks
        eff = t / (-(-t // sms) * sms)
        if eff > best_eff + 1e-9:
            best_eff, best = eff, ks
        ks += 1
    return min(best, nkb)


def mn_splits(nkb, k_splits):
    """The K-block ranges [lo, hi) of the k_splits splits of nkb K-blocks, as gemm_bf16_kernel divides them."""
    return [(ks * nkb // k_splits, (ks + 1) * nkb // k_splits) for ks in range(k_splits)]


# ------------------------------------------------------------------------------------------------- accumulator
def pad_k(t, mult=KB):
    """Zero-pad the columns of t (rows, K) to a multiple of `mult` (the TMA zero fill of a K tail)."""
    K = t.shape[1]
    Kp = -(-K // mult) * mult
    return t if Kp == K else torch.nn.functional.pad(t, (0, Kp - K))


def with_tail(a, w, ta, tw):
    """The K order of the LoRA tail: [A | 0 ..| tail_a | 0 ..] and [W | 0 ..| tail_w | 0 ..], each part padded to K-blocks."""
    return torch.cat([pad_k(a), pad_k(ta)], 1), torch.cat([pad_k(w), pad_k(tw)], 1)


def accumulate(a, w, k_splits=1, budget=1 << 28):
    """Exact acc = a w^T (float64) and its step slack for a (M, K), w (N, K) float64 holding bf16 values, K in the kernel's
    order.  k_splits > 1: also returns sum_ks |partial_ks| (the split-K reduce-add slack's weight), else None.  Rows are
    processed in chunks so that the (steps, rows, N) group sums stay within `budget` bytes."""
    a, w = pad_k(a), pad_k(w)
    M, Kp = a.shape
    N = w.shape[0]
    S = Kp // KSTEP
    wt = w.reshape(N, S, KSTEP).permute(1, 2, 0).contiguous()                   # (S, 16, N)
    splits = [(lo * 4, hi * 4) for lo, hi in mn_splits(Kp // KB, k_splits)]
    acc = torch.zeros(M, N, dtype=torch.float64, device=a.device)
    slack = (a.abs() @ w.abs().T) * U_ACC
    parts = torch.zeros_like(acc) if k_splits > 1 else None
    rows = max(1, budget // (S * N * 8))
    for r0 in range(0, M, rows):
        r1 = min(M, r0 + rows)
        g = torch.bmm(a[r0:r1].reshape(r1 - r0, S, KSTEP).permute(1, 0, 2), wt)  # (S, rows, N): group sums
        for s0, s1 in splits:
            c = g[s0:s1]
            c.cumsum_(0)
            p = c[-1].clone()
            acc[r0:r1] += p
            if parts is not None:
                parts[r0:r1] += p.abs()
            if s1 - s0 > 1:
                slack[r0:r1] += U_ACC * c[:-1].abs_().sum(0)
        del g
    return acc, slack, parts


def im2col(x, r0, r1):
    """Rows [r0, r1) of the implicit-GEMM operand of a 3x3 / pad 1 convolution over x (B, H, W, Cin) float64: row (b, y, x),
    columns (tap = 3 dy + dx, c) -- the kernel's tap-major K order."""
    B, H, W, Cin = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))
    idx = torch.arange(r0, r1, device=x.device)
    b, yy, xx = idx // (H * W), (idx // W) % H, idx % W
    cols = [xp[b, yy + dy, xx + dx] for dy in range(3) for dx in range(3)]
    return torch.cat(cols, 1)


def conv_accumulate(x, w, rows=4096):
    """accumulate() of the 3x3 convolution: x (B, H, W, Cin), w (Cout, 3, 3, Cin) float64; acc / slack (B H W, Cout)."""
    B, H, W, Cin = x.shape
    wk = w.reshape(w.shape[0], 9 * Cin)
    M = B * H * W
    accs, slacks = [], []
    for r0 in range(0, M, rows):
        acc, s, _ = accumulate(im2col(x, r0, min(M, r0 + rows)), wk)
        accs.append(acc)
        slacks.append(s)
    return torch.cat(accs), torch.cat(slacks)


# ------------------------------------------------------------------------------------------------- epilogues
def bias_out(acc, s_acc, bias):
    """y = acc + bias (fp32 add) and its slack."""
    y = acc if bias is None else acc + bias
    return y, s_acc + U * y.abs()


def gelu_out(y, s_y):
    """gelu(y) and the slack next to the GELU's 1-ulp contract; also |gelu'(y)| for callers that propagate it."""
    g, dg, _ = gelu64(y)
    return g, (dg.abs() + GELU2 * s_y) * s_y + GELU_TINY


def dgelu_out(acc, s_acc, pre):
    """acc gelu'(pre) and its slack; below 2^-40 the derivative's contract is absolute (its ex2 / rcp flush to zero)."""
    _, d, dt = gelu64(pre)
    return acc * d, d.abs() * s_acc + DGELU * acc.abs() * dt + GELU_TINY


def residual_out(y, s_y, gate, r, bf16=False):
    """out = r + gate y (the fmaf); bf16=True adds the fp32 rounding before the bf16 store."""
    o = r + gate * y
    s = gate.abs() * s_y
    return o, (s + U * o.abs()) if bf16 else s


def aux_out(val, s_val, scale=None):
    """aux = bf16(val [* scale]) of an fp32 value `val` with slack s_val (which must include val's own fp32 rounding)."""
    if scale is None:
        return val, s_val
    v = val * scale
    return v, scale.abs() * s_val + U * v.abs()


def f32_total(ref, s):
    """The slack of an fp32 output, its own half-ulp rounding included: what a value copied from it carries."""
    return s + 0.5 * f32_ulp(ref.abs() + s)


def row_stats_ref(out, BN):
    """float64 (sum o, sum o^2) per (row, column tile) of the fp32 `out` (M, N) the kernel wrote, their slacks (M, parts, 2)
    and the number of parts in use."""
    M, N = out.shape
    parts = -(-N // BN)
    o = torch.nn.functional.pad(out.double(), (0, parts * BN - N)).reshape(M, parts, BN)
    ref = torch.stack([o.sum(2), (o * o).sum(2)], 2)
    slack = torch.stack([(BN // 16 + 4) * U * o.abs().sum(2), (BN // 8 + 4) * U * (o * o).sum(2)], 2)
    return ref, slack, parts


def ln_prepare_ref(x, mult):
    """pxa_ln_prepare: a = x mult (x (M, C), mult broadcast per row) and its slack; stats (M, 2) = (sum x, sum x^2) and
    their slacks."""
    a = x * mult
    st = torch.stack([x.sum(1), (x * x).sum(1)], 1)
    s_st = torch.stack([16 * U * x.abs().sum(1), 41 * U * (x * x).sum(1)], 1)
    return a, U * a.abs(), st, s_st


def ln_epilogue_ref(acc, s_acc, stats, u, v, dim, eps):
    """EPI_LN_BIAS pre-activation x = rstd (acc - mu u) + v in float64 from the kernel's inputs: stats (M, 8, 2) fp32 parts,
    u / v (M, N) per row (the row's sample), and its slack (module docstring)."""
    sp, qp = stats[:, :, 0], stats[:, :, 1]
    S, Q = sp.sum(1, keepdim=True), qp.sum(1, keepdim=True)
    mu = S / dim
    q = Q / dim
    var = (q - mu * mu).clamp(min=0)
    rstd = 1 / torch.sqrt(var + eps)
    c = -rstd * mu
    x = rstd * acc + c * u + v
    e_mu = 3 * U * mu.abs() + 8 * U * sp.abs().sum(1, keepdim=True) / dim
    e_q = 3 * U * q + 8 * U * qp.abs().sum(1, keepdim=True) / dim
    e_var = e_q + 2 * mu.abs() * e_mu + U * mu * mu + U * var + U * (var + eps)
    rel = e_var / (2 * (var + eps)) + RSQRT
    e_c = c.abs() * (U + rel) + rstd * e_mu
    s = rstd * s_acc + rel * rstd * acc.abs() + e_c * u.abs() + U * (c * u + v).abs() + U * x.abs()
    return x, s


# ------------------------------------------------------------------------------------------------- tally
class Tally:
    """Accumulates |got - ref| / bound with bound = c ulp(|ref| + slack) + slack (bf16 or fp32 ulps) over the pieces of one
    output family; `check` prints the largest ratio, the fraction of elements equal to ref rounded to the output dtype and
    the bias statistic over |ref| > tiny, and asserts both."""

    def __init__(self, name, fp32=False, c=0.5, tiny=0.0):
        self.name, self.fp32, self.c, self.tiny = name, fp32, c, tiny
        self.worst, self.n, self.rounded, self.bias_sum, self.bias_n, self.bad = 0.0, 0, 0, 0.0, 0, 0
        self.example = None

    def add(self, got, ref, slack):
        got, ref = got.double(), ref.double()
        slack = torch.as_tensor(slack, dtype=torch.float64, device=ref.device).expand_as(ref)
        assert torch.isfinite(got).all(), f"{self.name}: {(~torch.isfinite(got)).sum().item()} non-finite results"
        ulp = f32_ulp if self.fp32 else bf16_ulp
        bound = self.c * ulp(ref.abs() + slack) + slack
        err = got - ref
        r = err.abs() / bound
        self.worst = max(self.worst, r.max().item())
        self.n += ref.numel()
        self.rounded += (got == ref.to(torch.float32 if self.fp32 else torch.bfloat16).double()).sum().item()
        big = ref.abs() > self.tiny
        self.bias_sum += (torch.sign(ref) * err / bound)[big].sum().item()
        self.bias_n += big.sum().item()
        bad = r > 1
        self.bad += bad.sum().item()
        if self.example is None and bad.any():
            i = torch.nonzero(bad.flatten())[:3, 0]
            self.example = (got.flatten()[i].tolist(), ref.flatten()[i].tolist(), bound.flatten()[i].tolist())
        return self

    @property
    def bias(self):
        return self.bias_sum / max(self.bias_n, 1)

    def max_bias(self):
        """MAX_BIAS for bf16 outputs; fp32 outputs are never rounded by a store, and their statistic shows the accumulator's
        own pull towards zero (module docstring), held only by the element-wise bound (|bias| <= 1)."""
        return 1.0 if self.fp32 else MAX_BIAS

    def ok(self):
        return self.bad == 0 and abs(self.bias) <= self.max_bias()

    def report(self, verbose=True):
        if verbose:
            print(f"{self.name}: {self.n} elements, max err / bound {self.worst:.3f}, correctly rounded "
                  f"{self.rounded / max(self.n, 1):.4f}, bias {self.bias:+.4f}, outside the bound {self.bad}")
        return self.worst, self.bias

    def check(self):
        worst, bias = self.report()
        max_bias = self.max_bias()
        assert self.bad == 0, f"{self.name}: {self.bad} elements outside the bound, e.g. got / want / bound {self.example}"
        assert abs(bias) <= max_bias, f"{self.name}: bias {bias:+.4f}"
        return worst, bias
