"""CPU emulations (numpy float32) of the kernels' GELU and GroupNorm-statistics formulas against float64.

They show that the element-wise contracts the GPU tests in test_numerics_gpu.py hold the kernels to are attainable in fp32,
and that the same contracts reject the formulas the kernels used before (so the bounds are not tuned to the kernels):

- GELU(tanh) and its derivative: within 1 bf16 ulp of the float64 value wherever |ref| > 2^-40, |result| <= 2^-40 elsewhere;
  the derivative gets 2^-20 (|s| + |2 x s (1 - s) u'|) of extra slack (the fp32 rounding of its two terms).
- GroupNorm statistics: the variance of a 4 M-element group with |mean| / std = 128 from fp32 sums.
"""
import numpy as np
import pytest
import torch

K0, K1 = 0.7978845608028654, 0.044715
TINY = 2.0 ** -40


def all_finite_bf16() -> np.ndarray:
    """Every finite bf16 value (both zeros, the subnormals), as float32."""
    bits = (np.arange(1 << 16, dtype=np.uint32) << 16).view(np.float32)
    return bits[np.isfinite(bits)]


def to_bf16(x32: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even to bf16, returned as float64 (what the kernels store)."""
    return torch.from_numpy(np.ascontiguousarray(x32, dtype=np.float32)).to(torch.bfloat16).double().numpy()


def bf16_ulp(ref: np.ndarray) -> np.ndarray:
    """The spacing of bf16 numbers at |ref| (8 significant bits; subnormal spacing 2^-133 below 2^-126)."""
    _, e = np.frexp(np.abs(ref))
    return np.ldexp(1.0, np.maximum(e - 8, -133))


def gelu64(x: np.ndarray):
    """float64 GELU(tanh) as x * sigmoid(2u) (== 0.5 x (1 + tanh u) exactly, without the cancellation of 1 + tanh u that
    costs even float64 its accuracy below x = -6), its derivative, and the derivative's two terms."""
    x = x.astype(np.float64)
    with np.errstate(over="ignore", divide="ignore"):
        u = K0 * (x + K1 * x ** 3)
        du = K0 * (1 + 3 * K1 * x * x)
        e = np.exp(-2 * u)
        s = 1 / (1 + e)
        t2 = 2 * x * (1 / (1 + 1 / e)) * du                   # 1 - s = e / (1 + e), also where e overflows
    return x * s, s + s * t2, np.abs(s) + np.abs(s * t2)


def violations(got: np.ndarray, ref: np.ndarray, slack=0.0) -> np.ndarray:
    """Mask of elements outside the contract: |got - ref| <= ulp(ref) + slack where |ref| > 2^-40, |got| <= 2^-40 + slack
    elsewhere (a non-finite result for a finite reference is outside)."""
    big = np.abs(ref) > TINY
    with np.errstate(invalid="ignore"):
        err = np.abs(got - ref)
        return ~np.isfinite(got) | np.where(big, err > bf16_ulp(ref) + slack, np.abs(got) > TINY + slack)


def _f32(v):
    return np.float32(v)


def gelu_tanh_form(x, tanh_rel=0.0):
    """The old kernel formula in float32, 0.5 x (1 + t), with t = tanh(u) off by tanh_rel (relative)."""
    x = x.astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        u = _f32(K0) * x * (_f32(K1) * x * x + _f32(1))
        t = (np.tanh(u) * _f32(1 + tanh_rel)).astype(np.float32)
        t = np.clip(t, -1, 1)
        du = _f32(K0) * (_f32(3 * K1) * x * x + _f32(1))
        return _f32(0.5) * x * (_f32(1) + t), _f32(0.5) * (_f32(1) + t) + _f32(0.5) * x * (_f32(1) - t * t) * du


def gelu_sigmoid_form(x, exp_rel=0.0):
    """The kernel formula in float32 (ptx.cuh gelu_tanh / gelu_tanh_grad): e = exp(-2u) off by exp_rel, s = 1 / (1 + e),
    gelu = x s; gelu' = s (1 + 2 xc min(e s, 1) u') on xc = x clamped to [-100, 100]."""
    x = x.astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        u = _f32(K0) * x * (_f32(K1) * x * x + _f32(1))
        e = (np.exp(_f32(-2) * u) * _f32(1 + exp_rel)).astype(np.float32)
        fwd = x * (_f32(1) / (_f32(1) + e))
        xc = np.clip(x, _f32(-100), _f32(100))
        uc = _f32(K0) * xc * (_f32(K1) * xc * xc + _f32(1))
        du = _f32(K0) * (_f32(3 * K1) * xc * xc + _f32(1))
        e = (np.exp(_f32(-2) * uc) * _f32(1 + exp_rel)).astype(np.float32)
        s = _f32(1) / (_f32(1) + e)
        es = np.fmin(e * s, _f32(1))
        return fwd, s * (_f32(2) * xc * es * du + _f32(1))


@pytest.mark.parametrize("exp_rel", [0.0, 2.0 ** -21, -(2.0 ** -21)])
def test_sigmoid_form_meets_the_gelu_contract_over_every_bf16_value(exp_rel):
    """x * sigmoid(2u) in float32 with exp(-2u) off by up to 2^-21 (ex2.approx.ftz is documented to about 2^-22; the fp32
    argument adds its own rounding) keeps every finite bf16 input inside the contract, forward and derivative."""
    x = all_finite_bf16()
    ref, dref, dterms = gelu64(x)
    fwd, grad = gelu_sigmoid_form(x, exp_rel)
    bad_f = violations(to_bf16(fwd), ref)
    bad_g = violations(to_bf16(grad), dref, 2.0 ** -20 * dterms)
    err_ulp = np.abs(to_bf16(fwd) - ref)[np.abs(ref) > TINY] / bf16_ulp(ref[np.abs(ref) > TINY])
    print(f"sigmoid form, exp off by {exp_rel:+.2e}: forward max {err_ulp.max():.3f} ulp, "
          f"{bad_f.sum()} / {bad_g.sum()} forward / derivative inputs outside the contract")
    assert not bad_f.any(), x[bad_f][:10]
    assert not bad_g.any(), x[bad_g][:10]


def test_tanh_form_fails_the_gelu_contract():
    """0.5 x (1 + tanh u) misses the same contract: with an exact float32 tanh for x in about [-6.4, -4.3] (256 ulp), and with
    tanh off by its documented 2^-11 (tanh.approx.f32) for hundreds of inputs down to x = -1.45, forward and derivative."""
    x = all_finite_bf16()
    ref, dref, dterms = gelu64(x)
    fwd, grad = gelu_tanh_form(x)
    bad_exact = violations(to_bf16(fwd), ref)
    worst_f, worst_g = np.zeros_like(bad_exact), np.zeros_like(bad_exact)
    for rel in (2.0 ** -11, -(2.0 ** -11)):
        f, g = gelu_tanh_form(x, rel)
        worst_f |= violations(to_bf16(f), ref)
        worst_g |= violations(to_bf16(g), dref, 2.0 ** -20 * dterms)
    near = worst_f & (np.abs(x) < 8)       # the model keeps the 2^-11 error where tanh.approx may well return -1 exactly
    print(f"tanh form: exact tanh {bad_exact.sum()} forward misses (x in [{x[bad_exact].min()}, {x[bad_exact].max()}]); "
          f"tanh off by 2^-11: {near.sum()} forward misses with |x| < 8 (x in [{x[near].min()}, {x[near].max()}]), "
          f"{(worst_g & (np.abs(x) < 8)).sum()} derivative misses")
    assert bad_exact.sum() > 20 and x[bad_exact].max() < -4
    assert near.sum() > 200 and x[near].max() > -1.6
    assert (worst_g & (np.abs(x) < 8)).sum() > 200


def test_gelu64_reference_equals_the_tanh_definition_where_float64_is_accurate():
    """The float64 sigmoid form is the tanh definition: equal to 1e-12 relative for x > -3, where 1 + tanh u > 2e-3 keeps all
    but 9 bits of float64."""
    x = np.linspace(-3, 8, 10001)
    ref, dref, _ = gelu64(x)
    u = K0 * (x + K1 * x ** 3)
    t = np.tanh(u)
    want = 0.5 * x * (1 + t)
    dwant = 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * K0 * (1 + 3 * K1 * x * x)
    assert np.allclose(ref, want, rtol=1e-12, atol=1e-300)
    assert np.allclose(dref, dwant, rtol=1e-10, atol=1e-14)


def _group_variance_fp32(x: np.ndarray, pivot: float) -> float:
    """fp32 one-pass statistics of the kernel's shape: 4096 sequential partial sums of x - pivot and (x - pivot)^2, combined
    sequentially, then var = E[d^2] - E[d]^2."""
    d = (x - np.float32(pivot)).astype(np.float32).reshape(4096, -1)
    s = np.cumsum(np.cumsum(d, axis=1, dtype=np.float32)[:, -1], dtype=np.float32)[-1]
    q = np.cumsum(np.cumsum(d * d, axis=1, dtype=np.float32)[:, -1], dtype=np.float32)[-1]
    n = np.float32(d.size)
    mean = s / n
    return float(max(q / n - mean * mean, np.float32(0)))


@pytest.mark.parametrize("ratio", [4, 32, 128, 512])
def test_pivoted_group_statistics_survive_large_offsets(ratio):
    """gn_stats_kernel sums x - K (K: the group's first element).  One-pass fp32 statistics of a 4 M-element group lose the
    variance to cancellation at |mean| / std = 128 (relative error > 1e-2); with the pivot they stay below 1e-4."""
    rng = np.random.default_rng(ratio)
    x = to_bf16((ratio + rng.standard_normal(1 << 22)).astype(np.float32))
    want = float(np.var(x))
    one_pass = abs(_group_variance_fp32(x, 0.0) - want) / want
    pivoted = abs(_group_variance_fp32(x, float(x[0])) - want) / want
    print(f"mean/std {ratio}: variance relative error one-pass {one_pass:.2e}, pivoted {pivoted:.2e}")
    assert pivoted < 1e-4
    if ratio >= 128:
        assert one_pass > 1e-2
