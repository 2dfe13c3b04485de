"""Float64 references and element-wise error bounds for one step of the optimizer kernels: the CAME step (pxa_came_flat,
optim_sm90.cu), AdamW (pxa_adamw_flat, elementwise_sm100.cu) and gradient-norm clipping (pxa_grad_clip_flat, optim_sm90.cu).
Shared by test_optim_numerics_cpu.py, which checks the bounds against a float32 emulation of the kernels, and
test_optim_numerics_gpu.py, which checks the kernels against them.

Each reference starts from the exact fp32 state the kernel started from (float64 tensors holding fp32 values) and takes ONE
step, so errors do not compound and every bound stays a few fp32 ulps wide.  Every output o is checked as
    |o_kernel - o_ref| <= 1/2 ulp32(|o_ref| + slack) + slack,
the half ulp for the final rounding to fp32, `slack` a first-order bound on everything before it, carried through the step
value by value as an absolute error e(.) in float64.  u = 2^-24 is the fp32 unit roundoff.  The terms, in the kernels' order:
  - roundings: every fp32 product, sum and quotient adds u |result|.  a * b + c * d may be contracted into an fma (nvcc's
    default --fmad=true); the bound of the unfused form covers both.  Products in the subnormal range (g ~ 1e-20 squared) add
    2^-150 absolute: the build does not flush denormals.
  - sums of n fp32 terms: (depth) u sum|x_i|, with depth the number of additions on the longest path of the kernel's order.
    CAME kind 2 (128 x 128 tiles): a row sum is 4 columns per lane + a 5-level shuffle tree + `coltiles` partials in
    came_finalize_kernel; a column sum is 16 rows per warp + 8 warp partials + `rowtiles` partials; the row mean of the
    statistics is ceil(R / 256) per thread + block_sum (5 + 8).  Kind 1 (matrices of at most 4 x 4, one per thread): R or C
    sequential additions.  The sums of u^2 (clip divisor) and of p^2 (rms) are per-thread fmaf chains (8 elements for 1-D
    tiles, R C for kind 1, 64 for kind 2) + block_sum + the fixed-order reduction of the tile sums.
  - rsqrtf: 2 ulp, 2^-22 relative (CUDA C Programming Guide, mathematical functions, without -use_fast_math, which build.py
    does not pass); an input error e(x) adds e(x) / (2 x) relative.  sqrtf is correctly rounded (u).
  - the CAME clip divisor max(RMS(u) / clip, 1): sqrtf of the sum of numel squares, the fp32 sqrt(numel) and two divisions.
    max(., 1) is 1-Lipschitz, so the divisor's error is that of RMS(u) / clip on either side of the kink.
  - d = u - m and res = d^2 + eps2: the errors of u and m are carried as absolute terms, so the cancellation in d costs what
    it costs (e(d) = e(u) + e(m) + u |d|, however small d is).
  - the division by the row mean rm, the update rf cf m lr and the weight decay p + (-wd lr) p: fp32(wd), -wd lr and its
    product with p each round, 3u |wd lr p|, and so does the sum.
  - clipping: the norm against float64 with the depth of its fmaf chains and trees (clip_norm_reference); every clipped
    gradient against (g grad_scale) coef with coef formed in fp32 from the norm the kernel computed, so that check is an
    ulp-level one of grad_clip_scale_kernel's own arithmetic (clip_bucket_reference).
The EMA coefficients are the fp32 numbers the kernels multiply by: b = fp32(beta) and omb = fp32(1 - beta), the difference
taken in double.  No fp32 kernel can multiply by 0.999 itself, and fp32(1 - beta) is what separates a correct kernel from one
forming 1.0f - fp32(beta) (1.3e-5 relative off at beta 0.999).  AdamW's bias corrections 1 - beta^t come from the double
betas as the caller gave them, as torch.optim.AdamW takes them; its decay factor is fp32(1 - lr wd), which torch's fp32
p.mul_(1 - lr wd) multiplies by as well (1 - 3e-6 is 0.4 ulp of p away from it, the same way for every element).

Bias: `Tally` reports two means over the elements, normalised by the bound: mean(sign(D) err / bound), D the reference's
change of that output in the step (the update of p, of exp_avg, of a statistic), and mean(sign(ref) err / bound).  A biased
coefficient (1.0f - beta, a bias correction of the fp32 beta, a row mean from stale statistics) pushes every error along D;
rounding toward zero pushes every error towards -sign(ref).  Either stays inside a worst-case bound element by element and
moves its mean.
"""
import math

import torch

U = 2.0 ** -24
RSQRT = 2.0 ** -22
TINY = 2.0 ** -150
MAX_BIAS = 0.05          # over >= MIN_BIAS_N elements; the correct emulation stays within ~0.03, the defects reach 0.1 .. 1
MIN_BIAS_N = 2000        # elements (and distinct |change|s) below which the mean is noise (err / bound spreads over +-1)

# pxa_came_flat's tiling (optim_sm90.cu)
THREADS, WARPS = 256, 8
VEC_TILE, SMALL_TILE, SMALL_MAX, TR, TC = 2048, 256, 4, 128, 128
BLOCK_SUM = 5 + WARPS
CLIP_PARTS = 1024


def f32(x):
    """x rounded to fp32, as a Python float."""
    return float(torch.tensor(float(x), dtype=torch.float64).float())


def f32_ulp(ref):
    """The spacing of fp32 numbers at |ref| (float64): 2^(e - 24) for |ref| in [2^(e-1), 2^e), 2^-149 below the normals."""
    _, e = torch.frexp(ref.abs())
    e = torch.where(ref == 0, torch.full_like(e, -125), e)           # frexp(0) has exponent 0
    return torch.ldexp(torch.ones_like(ref), (e - 24).clamp(min=-149))


def came_geom(shape):
    """(kind, lead, R, C, tiles) of a parameter of `shape`, as came_geom in optim_sm90.cu plans it."""
    n = math.prod(shape)
    if len(shape) < 2:
        return 0, 1, 1, n, -(-n // VEC_TILE)
    R, C = shape[-2], shape[-1]
    lead = n // (R * C)
    if R <= SMALL_MAX and C <= SMALL_MAX:
        return 1, lead, R, C, -(-lead // SMALL_TILE)
    return 2, lead, R, C, lead * -(-R // TR) * -(-C // TC)


def _sum(x, ex, dim, depth):
    """fp32 sum of x (>= 0) along dim in a tree of the given depth: value, error."""
    s = x.sum(dim)
    return s, ex.sum(dim) + depth * U * s


def _ema(old, b, omb, mean, e_mean):
    """b old + omb mean, rounded: value, error (old is exact)."""
    new = b * old + omb * mean
    return new, U * b * old.abs() + omb * (e_mean + U * mean.abs()) + U * new.abs()


def _factors(row, e_row, col, e_col, d_rm):
    """rsqrt(row / mean_R row) rsqrt(col) (lead, R, C) and its error, from the updated statistics (lead, R) / (lead, C)."""
    R = row.shape[-1]
    rm, e_rm = _sum(row, e_row, -1, d_rm)
    rm, e_rm = rm / R, e_rm / R + U * rm / R
    rm, e_rm = rm[..., None], e_rm[..., None]
    q = row / rm
    e_q = e_row / rm + row * e_rm / rm ** 2 + U * q
    rf = q.rsqrt()
    e_rf = rf * (0.5 * e_q / q + RSQRT)
    cf = col.rsqrt()
    e_cf = cf * (0.5 * e_col / col + RSQRT)
    f = rf[..., :, None] * cf[..., None, :]
    return f, e_rf[..., :, None] * cf[..., None, :] + rf[..., :, None] * e_cf[..., None, :] + U * f


def came_reference(p, g, m, state, *, lr, eps=(1e-30, 1e-16), clip_threshold=1.0, betas=(0.9, 0.999, 0.9999), weight_decay=0.0):
    """One CAME step (came_pytorch 0.1.3 semantics, include/pixart_sm100.h) of one parameter in float64, with the slack of
    every output.  p, g, m: float64 holding the fp32 parameter, gradient and exp_avg, in the parameter's shape; state: float64
    fp32 values of 'exp_avg_sq' (1-D) or 'exp_avg_sq_row' / '_col', 'exp_avg_res_row' / '_col' (came_pytorch's names and
    shapes); lr: the fp32 learning rate.  Returns {name: (ref, slack, change)} for 'param', 'exp_avg', the statistics and
    'RMS' (a 0-d tensor)."""
    shape = p.shape
    kind, lead, R, C, tiles = came_geom(tuple(shape))
    b1, b2, b3 = (f32(b) for b in betas)
    omb1, omb2, omb3 = (f32(1.0 - b) for b in betas)
    eps1, eps2, clip, wd = f32(eps[0]), f32(eps[1]), f32(clip_threshold), f32(weight_decay)
    n = p.numel()
    per_thread = {0: VEC_TILE // THREADS, 1: R * C, 2: (TR // WARPS) * (TC // 32)}[kind]
    d_tiles = BLOCK_SUM + -(-tiles // THREADS) + BLOCK_SUM
    d_row = {1: C, 2: TC // 32 + 5 + -(-C // TC)}.get(kind)
    d_col = {1: R, 2: TR // WARPS + WARPS + -(-R // TR)}.get(kind)
    d_rm = {1: R, 2: -(-R // THREADS) + BLOCK_SUM}.get(kind)
    out = {}

    x = g * g + eps1
    ex = 2 * U * x + TINY
    if kind == 0:
        v = state["exp_avg_sq"]
        v1, e_v1 = _ema(v, b2, omb2, x, ex)
        out["exp_avg_sq"] = (v1, e_v1, v1 - v)
        rv = v1.rsqrt()
        f, e_f = rv, rv * (0.5 * e_v1 / v1 + RSQRT)
    else:
        x3, ex3 = x.reshape(lead, R, C), ex.reshape(lead, R, C)
        sr, e_sr = _sum(x3, ex3, -1, d_row)
        sc, e_sc = _sum(x3, ex3, -2, d_col)
        row0, col0 = (state[k].reshape(lead, -1) for k in ("exp_avg_sq_row", "exp_avg_sq_col"))
        row, e_row = _ema(row0, b2, omb2, sr / C, e_sr / C + U * sr / C)
        col, e_col = _ema(col0, b2, omb2, sc / R, e_sc / R + U * sc / R)
        out["exp_avg_sq_row"] = (row, e_row, row - row0)
        out["exp_avg_sq_col"] = (col, e_col, col - col0)
        f, e_f = _factors(row, e_row, col, e_col, d_rm)
        f, e_f = f.reshape(shape), e_f.reshape(shape)
    u = f * g
    e_u = e_f * g.abs() + U * u.abs()

    s = (u * u).sum()
    e_s = (2 * u.abs() * e_u).sum() + (per_thread + d_tiles) * U * s
    a = s.sqrt() / math.sqrt(n) / clip
    e_a = a * (0.5 * e_s / s.clamp_min(1e-300) + 4 * U)
    div = a.clamp_min(1.0)
    uc = u / div
    e_uc = e_u / div + u.abs() * e_a / div ** 2 + U * uc.abs()

    m1, e_m1 = _ema(m, b1, omb1, uc, e_uc)
    out["exp_avg"] = (m1, e_m1, m1 - m)
    if kind == 0:
        upd, e_upd = m1, e_m1
    else:
        d = uc - m1
        e_d = e_uc + e_m1 + U * d.abs()
        r = d * d + eps2
        e_r = 2 * d.abs() * e_d + U * d * d + U * r + TINY
        r3, er3 = r.reshape(lead, R, C), e_r.reshape(lead, R, C)
        sr, e_sr = _sum(r3, er3, -1, d_row)
        sc, e_sc = _sum(r3, er3, -2, d_col)
        rrow0, rcol0 = (state[k].reshape(lead, -1) for k in ("exp_avg_res_row", "exp_avg_res_col"))
        rrow, e_rrow = _ema(rrow0, b3, omb3, sr / C, e_sr / C + U * sr / C)
        rcol, e_rcol = _ema(rcol0, b3, omb3, sc / R, e_sc / R + U * sc / R)
        out["exp_avg_res_row"] = (rrow, e_rrow, rrow - rrow0)
        out["exp_avg_res_col"] = (rcol, e_rcol, rcol - rcol0)
        f3, e_f3 = _factors(rrow, e_rrow, rcol, e_rcol, d_rm)
        f3, e_f3 = f3.reshape(shape), e_f3.reshape(shape)
        upd = f3 * m1
        e_upd = e_f3 * m1.abs() + f3 * e_m1 + U * upd.abs()
    step = upd * lr
    e_step = e_upd * lr + U * step.abs()
    decay = -wd * lr
    e_q = (3 * U * abs(decay) * p.abs() + U * (p + decay * p).abs()) if wd != 0 else torch.zeros_like(p)
    p1 = p - float(weight_decay) * lr * p - step
    out["param"] = (p1, e_q + e_step, p1 - p)

    sp = (p * p).sum()
    rms = sp.sqrt() / math.sqrt(n)
    d_p = per_thread + BLOCK_SUM + -(-tiles // 32) + 5
    out["RMS"] = (rms, rms * (0.5 * d_p * U + 3 * U), rms - rms)
    for k in [k for k in out if k.startswith(("exp_avg_sq_", "exp_avg_res_"))]:
        out[k] = tuple(t.reshape(state[k].shape) for t in out[k])
    return out


def adamw_reference(p, g, m, v, *, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, grad_scale=1.0):
    """One torch.optim.AdamW step (decoupled weight decay, bias corrections 1 - beta^step of the double betas) in float64,
    with slacks for pxa_adamw_flat: g' = g grad_scale; m = fmaf(b1, m, omb1 g'); v = fmaf(b2, v, (omb2 g') g');
    p = fmaf(-fp32(lr / bc1), m / (sqrtf(v) fp32(1 / sqrt(bc2)) + eps), p fp32(1 - lr wd)).  Returns {name: (ref, slack,
    change)} for 'param', 'exp_avg', 'exp_avg_sq'."""
    b1, b2 = f32(betas[0]), f32(betas[1])
    omb1, omb2 = f32(1.0 - betas[0]), f32(1.0 - betas[1])
    gs = f32(grad_scale)
    gk = g * gs
    e_gk = U * gk.abs() + TINY
    m1 = b1 * m + omb1 * gk
    e_m1 = omb1 * e_gk + U * omb1 * gk.abs() + U * m1.abs()
    v1 = b2 * v + omb2 * gk * gk
    e_v1 = omb2 * (2 * gk.abs() * e_gk + 2 * U * gk * gk) + U * v1 + TINY
    bc1, bc2 = 1.0 - betas[0] ** step, 1.0 - betas[1] ** step
    isb = 1.0 / math.sqrt(bc2)
    s = v1.sqrt()
    e_s = 0.5 * e_v1 / s.clamp_min(1e-300) + U * s
    den = s * isb + eps
    e_den = isb * e_s + 2 * U * s * isb + U * den + abs(f32(eps) - eps)
    r = m1 / den
    e_r = e_m1 / den + m1.abs() * e_den / den ** 2 + U * r.abs()
    delta = -(lr / bc1) * r
    e_delta = (lr / bc1) * e_r + U * delta.abs()
    decay = f32(1.0 - lr * weight_decay)
    e_decay = U * (p * decay).abs()
    p1 = p * decay + delta
    return {"param": (p1, e_delta + e_decay, p1 - p), "exp_avg": (m1, e_m1, m1 - m), "exp_avg_sq": (v1, e_v1, v1 - v)}


def clip_norm_reference(grads, lengths, *, grad_scale=1.0):
    """The 2-norm of the gradients after multiplying by grad_scale, in float64, with its slack for grad_sumsq_kernel /
    grad_clip_scale_kernel: each thread runs one fmaf chain over its float4s (stride 1024 x 256 threads) and tail element of
    every bucket, then block_sum, 4 partials per thread and block_sum again.  grads: the fp32 (or float64 holding fp32)
    buckets, converted one at a time; lengths: the elements of each bucket that are gradients.  Returns (norm, slack)."""
    gs = f32(grad_scale)
    ssq = sum(((g[:n].double() * gs) ** 2).sum() for g, n in zip(grads, lengths))
    chain = sum(4 * -(-(n // 4) // (CLIP_PARTS * THREADS)) + 1 for n in lengths)
    depth = chain + BLOCK_SUM + CLIP_PARTS // THREADS + BLOCK_SUM
    total = ssq.sqrt()
    return total, total * (0.5 * (depth + 2) * U + U)


def clip_bucket_reference(g, n, total, *, max_norm, grad_scale=1.0):
    """One bucket's clipped gradients given the norm `total` the kernel computed (checked on its own by
    clip_norm_reference): coef = fminf(fp32(max_norm) / (total + 1e-6f), 1.0f) formed in fp32 as grad_clip_scale_kernel forms
    it, then (g grad_scale) coef, whose only roundings are the two products.  Returns (clipped, slack, change)."""
    t = torch.tensor(float(total), dtype=torch.float32)
    coef = float(torch.clamp_max(torch.tensor(f32(max_norm), dtype=torch.float32) / (t + torch.tensor(1e-6, dtype=torch.float32)),
                                 1.0))
    g = g[:n].double()
    c = g * f32(grad_scale) * coef
    return c, U * c.abs() + TINY, c - g


class Tally:
    """Accumulates |got - ref| / bound with bound = 1/2 ulp32(|ref| + slack) + slack over the pieces of one output; `report`
    prints the largest ratio, the fraction of elements equal to ref rounded to fp32 and the two bias statistics."""

    def __init__(self, name):
        self.name = name
        self.worst, self.n, self.rounded, self.bias_sum, self.rbias_sum, self.bad = 0.0, 0, 0, 0.0, 0.0, 0
        self.distinct = 0
        self.example = None

    def add(self, got, ref, slack, change):
        got, ref, slack, change = (t.double().reshape(-1) for t in (got, ref, slack, change))
        assert torch.isfinite(got).all(), f"{self.name}: non-finite results"
        bound = 0.5 * f32_ulp(ref.abs() + slack) + slack
        err = got - ref
        r = err.abs() / bound
        self.worst = max(self.worst, r.max().item())
        self.n += ref.numel()
        self.distinct += torch.unique(change.abs().float()).numel()
        self.rounded += (got == ref.float().double()).sum().item()
        self.bias_sum += (torch.sign(change) * err / bound).sum().item()
        self.rbias_sum += (torch.sign(ref) * err / bound).sum().item()
        bad = r > 1
        self.bad += bad.sum().item()
        if self.example is None and bad.any():
            i = torch.nonzero(bad)[:3, 0]
            self.example = (got[i].tolist(), ref[i].tolist(), bound[i].tolist())
        return self

    def biased_enough(self):
        """Whether the bias statistics mean something: MIN_BIAS_N elements with as many distinct |change|.  Changes of one
        magnitude (CAME's first 1-D step is +-const) leave every element in a binade the same rounding error."""
        return min(self.n, self.distinct) >= MIN_BIAS_N

    def report(self, verbose=True):
        n = max(self.n, 1)
        bias, rbias = self.bias_sum / n, self.rbias_sum / n
        if verbose:
            print(f"{self.name}: {self.n} elements, max err / bound {self.worst:.3f}, correctly rounded {self.rounded / n:.4f}, "
                  f"bias along the change {bias:+.4f}, towards the value {rbias:+.4f}, outside the bound {self.bad}")
        return self.worst, bias, rbias

    def ok(self, max_bias=MAX_BIAS):
        _, bias, rbias = self.report(verbose=False)
        return self.bad == 0 and (not self.biased_enough() or (abs(bias) <= max_bias and abs(rbias) <= max_bias))

    def check(self, max_bias=MAX_BIAS):
        worst, bias, rbias = self.report()
        assert self.bad == 0, f"{self.name}: {self.bad} elements outside the bound, e.g. got / want / bound {self.example}"
        if self.biased_enough():
            assert abs(bias) <= max_bias and abs(rbias) <= max_bias, f"{self.name}: bias {bias:+.4f} / {rbias:+.4f}"
        return worst, bias, rbias


def mature_came_state(shape, seed, *, p_scale=0.02, g_scale=1e-3, zero=False):
    """fp32 (p, g, m, state) of one parameter for a CAME step from a mature state: gradients with row and column scales
    spread over 10x each around g_scale; row / column second-moment statistics that track those scales within +-20 %; exp_avg
    of the size of the normalised update (~0.3); instability statistics of the size of (u - m)^2 with spread; p at init scale
    (std p_scale).  zero: the state of step 1 (all statistics and exp_avg 0)."""
    gen = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    uni = lambda *s: torch.rand(*s, generator=gen, dtype=torch.float64)
    kind, lead, R, C, _ = came_geom(tuple(shape))
    sr = 10.0 ** (uni(lead, R, 1) - 0.5)
    sc = 10.0 ** (uni(lead, 1, C) - 0.5)
    g = (g_scale * sr * sc * rnd(lead, R, C)).reshape(shape)
    m = 0.3 * rnd(*shape)
    p = p_scale * rnd(*shape)
    jit = lambda *s: 0.8 + 0.4 * uni(*s)
    if kind == 0:
        state = {"exp_avg_sq": (g_scale * sr * sc).reshape(shape) ** 2 * jit(*shape)}
    else:
        lead_shape = tuple(shape[:-2])
        var = (g_scale * sr * sc) ** 2
        state = {"exp_avg_sq_row": (var.mean(-1) * jit(lead, R)).reshape(*lead_shape, R),
                 "exp_avg_sq_col": (var.mean(-2) * jit(lead, C)).reshape(*lead_shape, C),
                 "exp_avg_res_row": (jit(lead, R) ** 4).reshape(*lead_shape, R),
                 "exp_avg_res_col": (jit(lead, C) ** 4).reshape(*lead_shape, C)}
    if zero:
        m = torch.zeros_like(m)
        state = {k: torch.zeros_like(v) for k, v in state.items()}
    f = lambda t: t.float()
    return f(p), f(g), f(m), {k: f(v) for k, v in state.items()}


def mature_adamw_state(n, seed, *, p_scale=0.02, g_scale=1e-3, zero=False):
    """fp32 (p, g, m, v) of a flat AdamW bucket from a mature state: per-element gradient scales spread over 10x around
    g_scale, exp_avg ~ 0.3 of that scale, exp_avg_sq within +-20 % of its square.  zero: m = v = 0."""
    gen = torch.Generator().manual_seed(seed)
    s = g_scale * 10.0 ** (torch.rand(n, generator=gen, dtype=torch.float64) - 0.5)
    g = s * torch.randn(n, generator=gen, dtype=torch.float64)
    m = 0.3 * s * torch.randn(n, generator=gen, dtype=torch.float64)
    v = s ** 2 * (0.8 + 0.4 * torch.rand(n, generator=gen, dtype=torch.float64))
    p = p_scale * torch.randn(n, generator=gen, dtype=torch.float64)
    if zero:
        m, v = torch.zeros_like(m), torch.zeros_like(v)
    return p.float(), g.float(), m.float(), v.float()
