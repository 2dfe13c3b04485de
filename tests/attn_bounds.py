"""Float64 references and element-wise error bounds for the attention kernels: the head_dim-72 forward (attn_fwd.cuh, bf16 P
or bf16 hi + lo P), its backward (attn_bwd_sm90.cu) and the T5 forward (t5_attn_sm90.cu).  Shared by
test_attention_numerics_cpu.py, which checks the bounds against a float32 emulation of the kernels, and
test_attention_numerics_gpu.py, which checks the kernels against them.

Everything works on one (sample, head) at a time, with float64 tensors holding the bf16 (or fp32) inputs, on whatever device
they are on.  Notation: s_ij = q_i . k_j (exact in float64), c = scale log2(e), t_ij = c s_ij (+ log2(e) bias_ij for T5), the
logit in log2 units; m_i = max_j t_ij; P = softmax.  u = 2^-24 is the fp32 unit roundoff.

Forward, error of each unnormalised p_ij = exp2(t_ij - m) the kernel forms, relative (`eps`):
  - S = Q K^T accumulated in fp32 by wgmma: |dS_ij| <= D 2^-23 sum_d |q_id k_jd| (2^-23 per addition allows a truncating
    adder inside the tensor core);
  - scale_log2 = fp32(fp32(scale) fp32(log2 e)): 3u relative, i.e. 3u |t_ij| (T5 adds the bias in fp32 and multiplies by an
    fp32 log2 e: 3u log2(e) |bias_ij|);
  - the one rounding of fmaf(s, scale_log2, -m): u |t_ij - m_i|, plus u |t_ij| for the T5 kernel's separate product;
  - ex2.approx.ftz: 2^-22 relative (flushed results are below 2^-126 and vanish next to every term here);
  - corr = ex2(m_old - m_new) multiplies O and l alike, so its error is a relative error of the earlier keys' p: per block
    2^-22 + 2u (ex2, two products), plus ln2 u sum |m_old - m_new| = ln2 u (m_i - m_first_block_i) for the subtractions.
  The max itself cancels: every p and l are formed against the same fp32 m.
  A relative error eps_j of p_j moves o = sum p v / sum p by at most sum_j P_j eps_j (|v_jd| + |o_d|).
Forward output: slack_o = sum_j P_ij (eps_ij + rho + g_pv) |v_jd| + (sum_j P_ij eps_ij + g_l + 2u) |o_id|, plus one bf16 ulp
  for the final rounding, where
  - rho: P rounded to bf16 for P V, 2^-8 relative (an 8-bit significand, round to nearest); hi + lo P: 2^-16.  The
    normaliser l sums the unrounded fp32 p, so this error sits in the numerator alone;
  - g_pv = 2^-23 (16 + steps + nblk): the 16-product sum inside a k-step, one rounding of the fp32 accumulator per 16-key
    k-step (two with hi + lo P), one per block for the corr rescale;
  - g_l = u (blk/4 + 1) nblk + 2u: each thread sums blk/4 p per row and block, one fmaf with corr per block, two shuffles;
  - 2u: 1 / l and o * (1 / l).
lse = m + log2f(l) (fp32): m's own rounding cancels against l, leaving slack_lse = (sum_j P_ij eps_ij + g_l) / ln 2 + 2u |log2 l|
  (log2f, 1 ulp) + u |lse| (the sum), plus one fp32 ulp.

Backward, given the bf16 O and fp32 lse the forward produced:
  - Its contract is with the O and lse it is given: the reference delta_i = sum_d dO_id O_id uses that bf16 O in float64,
    and P* = exp2(t - lse*) is exact.  The kernel's P = ex2(fmaf(s, scale_log2, -lse)) then carries eps_b = ln2 (D 2^-23 c
    sum|q k| + 3u |t| + u |t - lse| + |lse - lse*|) + 2^-22: the lse error enters as what it is, measured, not bounded.
    (The gradient at the exact o* differs from this one by sum_d dO_id (O_id - o*_id) in delta, which the forward's contract
    bounds.)
  - dP = dO V^T in fp32: D 2^-23 sum_d |dO_id v_jd|; delta by attn_delta's fmaf chain: D u sum_d |dO_id O_id|.
  - dS = P (dP - delta) scale: three fp32 roundings (3u |dS|), then bf16 (2^-8 |dS|).  So
        |dS_kernel - dS*| <= E_ij = |dS*_ij| (eps_b + 3u + 2^-8) + (1 + 2^-8) P*_ij scale (dP error + delta error).
  - dQ = dS K, dK = dS^T Q, dV = P^T dO (P rounded to bf16, 2^-8) accumulated in fp32: 2^-23 (16 + n / 16) of sum |.| |.|
    over the n keys or queries.  Plus one bf16 ulp.
  slack_dq = E |K| + g sum_j |dS*_ij| |k_jd|,  slack_dk = E^T |Q| + g ...,  slack_dv = (P* (eps_b + 2^-8))^T |dO| + g ...
  With keys sharing an offset k_j = kbar + kappa_j, sum_j dS_ij = 0 cancels kbar out of the exact dQ, but the errors of dS do
  not cancel: E |K| contains |kbar_d| (scale P (delta error) + 2^-8 |dS|) summed over the keys, the residue the kernel must
  stay under.  Rounding delta to bf16 (2^-8 |delta|) instead of keeping it in fp32 breaks it many times over wherever |delta|
  is large next to |dP - delta| (25x with values and dO offset, in test_attention_numerics_cpu).

Bias: `Tally` also reports mean(sign(ref) (got - ref) / bound) over the elements.  Round to nearest leaves it at 0; rounding
toward zero (truncation) pulls every element's error towards -sign(ref) and makes it negative, while its error stays inside
any worst-case bound.  It is normalised by the bound rather than ulp(ref) because attention outputs have many small elements
whose ulp says nothing about their error scale.
"""
import math

import torch

from test_backward_numerics_gpu import f32_ulp
from test_numerics_gpu import bf16_ulp

U = 2.0 ** -24
U_ACC = 2.0 ** -23
EX2 = 2.0 ** -22
LN2 = math.log(2.0)
LOG2E = 1.4426950408889634
RHO_BF16 = 2.0 ** -8
RHO_HI_LO = 2.0 ** -16
MAX_BIAS = 0.05          # |mean(sign(ref) err / bound)|: round to nearest stays within 0.015, truncated P reaches -0.2 to -0.3


DISTRIBUTIONS = ["diffuse", "peaked", "peaked_rev", "offset_logits", "offset_vk"]


def make_inputs(name, lead, Nq, L, D, seed, device="cpu"):
    """bf16 q (*lead, Nq, D), k / v (*lead, L, D) and dO (*lead, Nq, D) as float64, for the named distribution:
      diffuse:       N(0, 1) everywhere; a near-uniform softmax over many keys;
      peaked:        q x 7 and key norms ramping from 0.3 to 1.2 along the keys, so the running max grows block by block and
                     every corr rescale fires (peaked_rev: the ramp reversed, the max sits in the first block);
      offset_logits: q and k share a +-4 direction, which puts every logit near 200 log2 units;
      offset_vk:     v = 4 + noise, k = kbar + noise (kbar one N(0, 1) vector), dO = 1 + noise."""
    g = torch.Generator(device=device).manual_seed(seed)
    n = lambda *s: torch.randn(*lead, *s, generator=g, dtype=torch.float64, device=device)
    q, k, v, do = n(Nq, D), n(L, D), n(L, D), n(Nq, D)
    if name.startswith("peaked"):
        ramp = torch.linspace(0.3, 1.2, L, dtype=torch.float64, device=device)[:, None]
        k = k * (ramp if name == "peaked" else ramp.flip(0))
        q = q * 7
    elif name == "offset_logits":
        u = torch.randint(0, 2, (D,), generator=g, device=device).double() * 2 - 1
        q, k = 4 * u + q, 4 * u + k
    elif name == "offset_vk":
        v = v + 4
        k = k + n(1, D)
        do = do + 1
    bf = lambda x: x.to(torch.bfloat16).double()
    return bf(q), bf(k), bf(v), bf(do)


def forward(q, k, v, scale, *, blk=128, split_p=False, bias=None):
    """float64 softmax(q k^T scale + bias) v of one (sample, head) and its bounds.  q (Nq, D), k / v (L, D): the valid keys
    only; bias (Nq, L) or None (T5: the fp32 bias in natural-log units, -inf or finfo.min where masked).  Returns a dict:
    o, lse (log2 units), slack_o, slack_lse, and what the backward bound reuses."""
    L, D = k.shape
    c = scale * LOG2E
    s = q @ k.T
    t = c * s
    dt = (c * D * U_ACC) * (q.abs() @ k.abs().T) + 3 * U * t.abs()
    if bias is not None:
        bias = bias.clamp(min=torch.finfo(torch.float32).min)
        t = t + LOG2E * bias
        dt = dt + 3 * U * LOG2E * bias.abs() + U * t.abs()
    m = t.max(1, keepdim=True).values
    e = torch.exp2(t - m)
    l = e.sum(1, keepdim=True)
    P = e / l
    o = P @ v
    lse = (m + torch.log2(l))[:, 0]
    nblk = -(-L // blk)
    m_first = t[:, :blk].max(1, keepdim=True).values
    corr = nblk * (EX2 + 2 * U) + LN2 * U * (m - m_first)
    eps = LN2 * (dt + U * (m - t)) + EX2 + corr
    Pe = P * eps
    Pe = torch.where(P > 0, Pe, torch.zeros_like(Pe))               # masked keys: P = 0 whatever the logit's size
    steps = (L / 16) * (2 if split_p else 1)
    g_pv = U_ACC * (16 + steps + nblk)
    g_l = U * ((blk // 4 + 1) * nblk + 2)
    rho = RHO_HI_LO if split_p else RHO_BF16
    pe_sum = Pe.sum(1, keepdim=True)
    slack_o = (Pe + (rho + g_pv) * P) @ v.abs() + (pe_sum + g_l + 2 * U) * o.abs()
    slack_lse = (pe_sum[:, 0] + g_l) / LN2 + 2 * U * torch.log2(l)[:, 0].abs() + U * lse.abs()
    return dict(o=o, lse=lse, slack_o=slack_o, slack_lse=slack_lse, P=P, t=t, dt=dt)


def backward(q, k, v, do, o, lse, scale, fwd=None):
    """float64 gradients of one (sample, head) and their bounds, for the backward given the bf16 forward output `o` (Nq, D)
    and the fp32 `lse` (Nq,) (see the module docstring).  k / v: the valid keys only.  `fwd`: forward(q, k, v, scale) if
    already computed.  Returns a dict: dq, dk, dv, slack_dq, slack_dk, slack_dv."""
    fwd = fwd or forward(q, k, v, scale)
    Nq, D = q.shape
    L = k.shape[0]
    P, t, dt = fwd["P"], fwd["t"], fwd["dt"]
    dlse = (lse - fwd["lse"]).abs()[:, None]
    eps = LN2 * (dt + U * (t - lse[:, None]).abs() + dlse) + EX2
    delta = (do * o).sum(1, keepdim=True)
    dP = do @ v.T
    dS = P * (dP - delta) * scale
    err_in = (D * U_ACC) * (do.abs() @ v.abs().T) + (D * U) * (do * o).abs().sum(1, keepdim=True)
    E = dS.abs() * (eps + 3 * U + RHO_BF16) + (1 + RHO_BF16) * scale * P * err_in
    aS = dS.abs()
    g_q = U_ACC * (16 + L / 16)
    g_kv = U_ACC * (16 + Nq / 16)
    return dict(dq=dS @ k, dk=dS.T @ q, dv=P.T @ do,
                slack_dq=E @ k.abs() + g_q * (aS @ k.abs()),
                slack_dk=E.T @ q.abs() + g_kv * (aS.T @ q.abs()),
                slack_dv=(P * (eps + RHO_BF16)).T @ do.abs() + g_kv * (P.T @ do.abs()))


class Tally:
    """Accumulates |got - ref| / bound, with bound = ulp(ref) + slack (bf16 ulps, or fp32 ulps for lse), over several
    (sample, head) pieces of one output; `report` prints the largest ratio, the fraction of elements equal to ref rounded to
    bf16 and the bias statistic, and returns them."""

    def __init__(self, name, fp32=False):
        self.name, self.fp32 = name, fp32
        self.worst, self.n, self.rounded, self.bias_sum, self.bad = 0.0, 0, 0, 0.0, 0
        self.example = None

    def add(self, got, ref, slack):
        got, ref = got.double(), ref.double()
        bound = (f32_ulp(ref) if self.fp32 else bf16_ulp(ref)) + slack
        err = got - ref
        r = err.abs() / bound
        assert torch.isfinite(got).all(), f"{self.name}: non-finite results"
        self.worst = max(self.worst, r.max().item())
        self.n += ref.numel()
        self.rounded += (got == ref.to(torch.bfloat16).double()).sum().item()
        self.bias_sum += (torch.sign(ref) * err / bound).sum().item()
        bad = r > 1
        self.bad += bad.sum().item()
        if self.example is None and bad.any():
            i = torch.nonzero(bad.flatten())[:3, 0]
            self.example = (got.flatten()[i].tolist(), ref.flatten()[i].tolist(), bound.flatten()[i].tolist())

    def report(self, verbose=True):
        bias = self.bias_sum / max(self.n, 1)
        if verbose:
            print(f"{self.name}: {self.n} elements, max err / bound {self.worst:.3f}, correctly rounded "
                  f"{self.rounded / max(self.n, 1):.4f}, bias {bias:+.4f}, outside the bound {self.bad}")
        return self.worst, bias

    def check(self, max_bias=MAX_BIAS):
        worst, bias = self.report()
        assert self.bad == 0, f"{self.name}: {self.bad} elements outside the bound, e.g. got / want / bound {self.example}"
        assert abs(bias) <= max_bias, f"{self.name}: bias {bias:+.4f}"
        return worst, bias
