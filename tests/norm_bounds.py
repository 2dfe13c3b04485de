"""Element-wise bounds of the LayerNorm kernels (ln_modulate, layernorm_affine_, ln_modulate_bwd and the LayerNorm inside
kv_compress_bwd), shared by test_numerics_gpu.py, test_backward_numerics_gpu.py and block_stages.py.  Pure float64 torch on
whatever device the tensors are on."""
import torch

U = 2.0 ** -24                      # fp32 unit roundoff


def ln_slack(xd, ratio_rows, mult):
    """fp32 two-pass LayerNorm: the mean is a sum of C terms in <= 64 sequential fp32 additions (per-lane runs, then a
    butterfly), so (x - mean) carries up to 2^-18 |mean| absolute error; relative to std that is 2^-18 |mean| / std, times
    the output multiplier."""
    return 2.0 ** -18 * (1 + ratio_rows) * mult


def ln_stats(xd, eps):
    mean = xd.mean(-1, keepdim=True)
    var = xd.var(-1, unbiased=False, keepdim=True)
    rstd = 1 / torch.sqrt(var + eps)
    return (xd - mean) * rstd, rstd, mean.abs() / var.sqrt().clamp(min=1e-30)


def ln_bwd_slack(xh, rstd, g, r, rstd_rel):
    """Element-wise bound on the fp32 error of dx = rstd (g - mean_c g - xh mean_c(g xh)) over the last dim, from float64
    xh, rstd, g = dxn (1 + scale) (or dy gamma) and r = |mean| / std of the row:
      - the kernel's xh carries e = 2^-18 (1 + r) (the row mean: a sum of C terms in <= 41 sequential fp32 additions, 36
        per lane then 5 butterfly levels, see ln_slack) + 2^-19 |xh| (rstd and the rounding of (x - mean) rstd); a
        perturbation e of xh moves dx by rstd (e |mean(g xh)| + |xh| mean(|g| e));
      - 3 rstd_rel T for the relative error of rstd, which enters dx, xh and mean(g xh) once each, and 2^-18 T for the
        roundings of g, of the two means (<= 41 additions each) and of the final expression, where
        T = rstd (|g| + mean|g| + |xh| mean|g xh|) bounds every term's magnitude."""
    mg, mgx = g.mean(-1, keepdim=True), (g * xh).mean(-1, keepdim=True)
    e = 2.0 ** -18 * (1 + r) + 2.0 ** -19 * xh.abs()
    T = rstd * (g.abs() + g.abs().mean(-1, keepdim=True) + xh.abs() * (g * xh).abs().mean(-1, keepdim=True))
    return (3 * rstd_rel + 2.0 ** -18) * T + rstd * (e * mgx.abs() + xh.abs() * (g.abs() * e).mean(-1, keepdim=True))


def sample_sum_slack(b_of, B, rpb, M, terms, pre):
    """Bound on the fp32 error of pre[b] + sum_{rows of b} terms: sequential runs of <= 16 rows per warp (<= 15 u sum|terms|),
    then one atomic per warp that touches sample b onto pre (W_b atomics: <= W_b u (|pre| + sum|terms|))."""
    first = torch.arange(B, device=terms.device) * rpb
    last = torch.clamp(first + rpb, max=M) - 1
    wb = (last // 16 - first // 16 + 1).double()[:, None]
    return (15 + wb) * U * (pre.double().abs() + torch.zeros_like(pre, dtype=torch.float64).index_add(0, b_of, terms.abs()))
