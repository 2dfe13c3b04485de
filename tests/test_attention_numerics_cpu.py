"""The attention bounds of attn_bounds.py checked against a float32 emulation of the kernels' arithmetic, on the CPU.

The emulation follows attn_fwd.cuh and attn_bwd_sm90.cu step by step at a few hundred queries and keys: 128-key blocks, the
running max and the corr rescale of O and l in every block, logits as fmaf(s, scale_log2, -m), l summed from the unrounded
fp32 p, P rounded to bf16 (or bf16 hi + lo) for P V, O / l rounded to bf16 and lse = m + log2 l; in the backward P from the
lse, delta from the bf16 O in fp32, dS = P (dP - delta) scale rounded to bf16.  The tests show that

- the correct emulation stays inside every bound on every distribution the GPU file uses, with a bias statistic near 0;
- defects of the size of the rounding itself are rejected: P truncated to bf16 instead of rounded (forward and dV), dS
  truncated, delta rounded to bf16, one block's corr skipped, the last block's key mask off by one;
- the normwise bounds the other attention tests use (6e-3 forward, 1e-2 backward) accept the first three of those defects,
  which is the gap the element-wise contract closes.

With -s every case prints its largest error / bound and bias.
"""
import math

import pytest
import torch

import attn_bounds as ab

D = 72
SCALE = D ** -0.5
F32 = torch.float32


def rn(x):
    return x.to(torch.bfloat16).float()


def rz(x):
    """bf16 rounding toward zero: the low 16 bits of the fp32 pattern dropped."""
    return (x.contiguous().view(torch.int32) & ~0xFFFF).view(F32)


def f32(x):
    return torch.tensor(x, dtype=F32)


def fma(a, b, c):
    """fmaf: one rounding of the exact a b + c (float64 holds the product of two fp32 values exactly)."""
    return (a.double() * b.double() + c.double()).float()


def emulate_forward(q, k, v, scale, *, split_p=False, defect=None, blk=128):
    """attn_fwd.cuh on one (sample, head): q (Nq, D), k / v (L, D) bf16 values.  Returns (bf16 O, fp32 lse) as float64.
    defect: "p_trunc" (P rounded toward zero), "corr" (block 1 skips its rescale), "mask" (the last block's mask drops the
    last valid key)."""
    qf, kf, vf = q.float(), k.float(), v.float()
    L = k.shape[0]
    sl2 = f32(scale) * f32(ab.LOG2E)
    S = qf @ kf.T
    Nq = q.shape[0]
    m = torch.full((Nq,), -math.inf, dtype=F32)
    l = torch.zeros(Nq, dtype=F32)
    o = torch.zeros(Nq, D, dtype=F32)
    nblk = -(-L // blk)
    for n in range(nblk):
        rem = min(blk, L - n * blk)
        if defect == "mask" and n == nblk - 1:
            rem -= 1
        Sb = S[:, n * blk:n * blk + rem]
        m_new = torch.maximum(m, Sb.max(1).values * sl2)
        corr = torch.exp2(m - m_new)
        if defect == "corr" and n == 1:
            corr = torch.ones_like(corr)
        p = torch.exp2(fma(Sb, sl2, -m_new[:, None]))
        l = fma(l, corr, p.sum(1))
        ph = rz(p) if defect == "p_trunc" else rn(p)
        o = o * corr[:, None] + ph @ vf[n * blk:n * blk + rem]
        if split_p:
            o = o + rn(p - ph) @ vf[n * blk:n * blk + rem]
        m = m_new
    return rn(o * (1.0 / l)[:, None]).double(), (m + torch.log2(l)).double()


def emulate_backward(q, k, v, do, o, lse, scale, *, defect=None):
    """attn_bwd_sm90.cu (and attn_delta) on one (sample, head).  Returns bf16 (dq, dk, dv) as float64.  defect: "p_trunc"
    (P truncated for dV), "ds_trunc" (dS truncated), "delta_bf16" (delta rounded to bf16)."""
    qf, kf, vf, dof = q.float(), k.float(), v.float(), do.float()
    sl2 = f32(scale) * f32(ab.LOG2E)
    P = torch.exp2(fma(qf @ kf.T, sl2, -lse.float()[:, None]))
    delta = (dof * o.float()).sum(1)
    if defect == "delta_bf16":
        delta = rn(delta)
    dS = P * (dof @ vf.T - delta[:, None]) * f32(scale)
    dSb = rz(dS) if defect == "ds_trunc" else rn(dS)
    Pb = rz(P) if defect == "p_trunc" else rn(P)
    return rn(dSb @ kf).double(), rn(dSb.T @ qf).double(), rn(Pb.T @ dof).double()


CASES = ab.DISTRIBUTIONS
NQ, L = 300, 330                              # 3 key blocks, the last partial; Nq not a multiple of 64


def run(name, *, split_p=False, fdef=None, bdef=None, heads=2):
    """Emulate forward and backward on `heads` (sample, head) pieces; returns {output: Tally} and normwise errors."""
    tal = {o: ab.Tally(f"{name} {o}", fp32=(o == "lse")) for o in ("o", "lse", "dq", "dk", "dv")}
    num, den = {o: 0.0 for o in tal}, {o: 0.0 for o in tal}
    for h in range(heads):
        q, k, v, do = ab.make_inputs(name, (), NQ, L, D, seed=7 * h + len(name))
        fw = ab.forward(q, k, v, SCALE, split_p=split_p)
        o, lse = emulate_forward(q, k, v, SCALE, split_p=split_p, defect=fdef)
        bw = ab.backward(q, k, v, do, o, lse, SCALE, fwd=fw)
        dq, dk, dv = emulate_backward(q, k, v, do, o, lse, SCALE, defect=bdef)
        for key, got, ref, sl in (("o", o, fw["o"], fw["slack_o"]), ("lse", lse, fw["lse"], fw["slack_lse"]),
                                  ("dq", dq, bw["dq"], bw["slack_dq"]), ("dk", dk, bw["dk"], bw["slack_dk"]),
                                  ("dv", dv, bw["dv"], bw["slack_dv"])):
            tal[key].add(got, ref, sl)
            num[key] += ((got - ref) ** 2).sum().item()
            den[key] += (ref ** 2).sum().item()
    return tal, {key: math.sqrt(num[key] / den[key]) for key in tal}


@pytest.mark.parametrize("split_p", [False, True])
@pytest.mark.parametrize("name", CASES)
def test_correct_emulation_meets_the_bounds(name, split_p):
    tal, _ = run(name, split_p=split_p)
    for t in tal.values():
        t.check()


def _rejected(tal, out):
    worst, bias = tal[out].report()
    return worst > 1 or abs(bias) > ab.MAX_BIAS


# (defect, distribution, the output whose contract must reject it): truncation by the bias statistic, where the errors pull
# one way (values and dO offset for P, the peaked softmax for dS); bf16 delta in dQ with keys sharing an offset.
DEFECTS = [("p_trunc", "offset_vk", "o"), ("p_trunc_dv", "offset_vk", "dv"), ("ds_trunc", "peaked", "dk"),
           ("delta_bf16", "offset_vk", "dq"), ("corr", "diffuse", "o"), ("mask", "diffuse", "o")]


@pytest.mark.parametrize("defect,case,out", DEFECTS)
def test_emulated_defects_are_rejected(defect, case, out):
    fdef = defect if defect in ("p_trunc", "corr", "mask") else None
    bdef = {"p_trunc_dv": "p_trunc", "ds_trunc": "ds_trunc", "delta_bf16": "delta_bf16"}.get(defect)
    tal, _ = run(case, fdef=fdef, bdef=bdef)
    assert _rejected(tal, out), f"{defect} passes the {out} contract"


@pytest.mark.parametrize("defect", ["p_trunc", "ds_trunc", "delta_bf16"])
def test_old_normwise_bounds_accept_rounding_sized_defects(defect):
    """The normwise bounds of test_attn_pipeline_gpu / test_backward_gpu (6e-3 for O, 1e-2 for dQ / dK / dV) on the same
    diffuse inputs they use pass all three defects, so only the element-wise contract and its bias statistic stand between
    them and the kernels."""
    _, nw = run("diffuse", fdef="p_trunc" if defect == "p_trunc" else None, bdef=defect)
    print(defect, {k_: f"{e:.2e}" for k_, e in nw.items()})
    assert nw["o"] < 6e-3 and max(nw["dq"], nw["dk"], nw["dv"]) < 1e-2
