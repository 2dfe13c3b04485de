"""The GEMM-family bounds of gemm_bounds.py are attainable and sharp (CPU only).

The kernels are emulated in float32 at small shapes that keep the structure that matters: K tails (K = 200), a LoRA tail
(T = 24), split-K weight gradients (3 splits) and a 3x3 convolution whose border taps read zero padding.  Two accumulator
models:
  (a) `seq`:   sequential fp32, one round-to-nearest addition per product in the kernel's K order;
  (b) `trunc`: per wgmma k16 step, the 16 products and the accumulator are aligned to the largest exponent, each truncated to
               24 bits there, summed exactly, and the sum truncated to fp32 (a truncating adder without guard bits).
Both must stay inside every bound with the bias statistic inside gemm_bounds.MAX_BIAS.  Ten defects, emulated on model (a),
must each be rejected; the test also prints whether the normwise checks used elsewhere in the suite (rel_err < 4e-3 for bf16
outputs, < 2e-4 for fp32 ones) would have accepted them.

MAX_BIAS: the two models stay within |bias| 0.008 on every family (the truncating model's own pull towards zero is a small
fraction of the accumulator slack), while a truncating bf16 store moves the bias of every stored family to -0.49 (GELU, whose
bound is 1 ulp) or about -1; 0.1 leaves a margin of more than 10x over the models and about 5x under the smallest defect
(printed by test_bias_threshold_separates, which asserts at least 3x and 2.5x).
"""
import pytest
import torch

import gemm_bounds as gb

pytestmark = pytest.mark.slow

BF = torch.bfloat16
F64 = torch.float64


def bf(x):
    return x.to(BF).double()


def bf_rz(x):
    """float64 -> fp32 (exact here) -> bf16 rounded toward zero, as float64."""
    b = x.float().contiguous().view(torch.int32) & -65536
    return b.view(torch.float32).double()


def f32(x):
    return x.float().double()


def f32_rz(x):
    r = x.float()
    over = r.double().abs() > x.abs()
    r = torch.where(over, torch.nextafter(r, torch.zeros_like(r)), r)
    return r.double()


def fma(a, b, c):
    return f32(a * b + c)


def randn(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=F64) * scale


# ------------------------------------------------------------------------------------------------- accumulator models
def acc_seq(a, w, k_splits=1, bf16_after_kb=None):
    """Model (a): sequential fp32 over the padded K order; returns the k_splits partial sums.  bf16_after_kb: round the
    accumulator to bf16 once, after that K-block (defect 8)."""
    a, w = gb.pad_k(a), gb.pad_k(w)
    out = []
    for lo, hi in gb.mn_splits(a.shape[1] // gb.KB, k_splits):
        acc = torch.zeros(a.shape[0], w.shape[0], dtype=F64)
        for k in range(lo * gb.KB, hi * gb.KB):
            acc = f32(acc + torch.outer(a[:, k], w[:, k]))
            if bf16_after_kb is not None and k == (bf16_after_kb + 1) * gb.KB - 1:
                acc = bf(acc)
        out.append(acc)
    return out


def acc_trunc(a, w, k_splits=1):
    """Model (b): truncating aligned 17-term adder per k16 step."""
    a, w = gb.pad_k(a), gb.pad_k(w)
    out = []
    for lo, hi in gb.mn_splits(a.shape[1] // gb.KB, k_splits):
        acc = torch.zeros(a.shape[0], w.shape[0], dtype=F64)
        for s in range(lo * 4, hi * 4):
            k = slice(s * gb.KSTEP, (s + 1) * gb.KSTEP)
            terms = torch.cat([a[:, None, k] * w[None, :, k], acc[..., None]], 2)
            _, e = torch.frexp(terms.abs().amax(2, keepdim=True))
            q = torch.ldexp(torch.ones_like(terms[..., :1]), e - 24)
            acc = f32_rz(torch.trunc(terms / q).sum(2, keepdim=True)[..., 0] * q[..., 0])
        out.append(acc)
    return out


MODELS = {"seq": acc_seq, "trunc": acc_trunc}


# ------------------------------------------------------------------------------------------------- cases
B, RPB, N, K, T, BN = 2, 80, 320, 200, 24, 128
M = B * RPB


def fwd_inputs():
    a = bf(randn(M, K, seed=1))
    w = bf(randn(N, K, seed=2, scale=K ** -0.5))
    w_gelu = bf(randn(N, K, seed=3, scale=3 * K ** -0.5))          # pre-activation std 3: the GELU's negative tail
    bias = bf(randn(N, seed=4, scale=0.1))
    ta, tw = bf(randn(M, T, seed=5)), bf(randn(N, T, seed=6, scale=0.5 * T ** -0.5))
    gate = f32(randn(B, N, seed=7)).repeat_interleave(RPB, 0)
    res = f32(randn(M, N, seed=8))
    scale = f32(1 + 0.3 * randn(B, N, seed=9)).repeat_interleave(RPB, 0)
    pre = bf(randn(M, N, seed=10, scale=3))
    return dict(a=a, w=w, w_gelu=w_gelu, bias=bias, ta=ta, tw=tw, gate=gate, res=res, scale=scale, pre=pre)


def row_stats_emul(o, bn, from_bf16=False, wrong_part=False, no_zero=False):
    """row_stats_out as the kernel forms it (pair sums, BN / 16 pairs per thread, 2 shuffle levels, two warpgroups)."""
    if from_bf16:
        o = bf(o)
    parts = -(-o.shape[1] // bn)
    op = torch.nn.functional.pad(o, (0, parts * bn - o.shape[1]))
    st = torch.full((o.shape[0], gb.LN_STAT_PARTS, 2), 1.0 if no_zero else 0.0, dtype=F64)       # 1.0: a stale value
    for t in range(parts):
        tile = op[:, t * bn:(t + 1) * bn].reshape(o.shape[0], 2, bn // 64, 4, 4, 2)   # (g, slab, jj, lane, pair)
        s = torch.zeros(o.shape[0], 2, 4, dtype=F64)
        q = torch.zeros_like(s)
        for sl in range(bn // 64):
            for jj in range(4):
                x0, x1 = tile[:, :, sl, jj, :, 0], tile[:, :, sl, jj, :, 1]
                s = f32(s + f32(x0 + x1))
                q = fma(x0, x0, fma(x1, x1, q))
        for v in (s, q):
            v.copy_(f32(v + v[:, :, [1, 0, 3, 2]]))
            v.copy_(f32(v + v[:, :, [2, 3, 0, 1]]))
        st[:, (t + 1) % parts if wrong_part else t] = torch.stack([f32(s[:, 1, 0] + s[:, 0, 0]), f32(q[:, 1, 0] + q[:, 0, 0])], 1)
    if not no_zero:
        st[:, parts:] = 0
    return st


def emulate_fwd(x, model, defect=None):
    """Every forward epilogue of one shape: {family: kernel output (float64)}."""
    store = bf_rz if defect == "rz_store" else bf
    acc_fn = MODELS[model]
    kw = dict(bf16_after_kb=1) if defect == "acc_bf16_between_kblocks" else {}
    acc = acc_fn(x["a"], x["w"], **kw)[0]
    if defect == "lora_tail_own_acc_bf16":
        acc_t = f32(acc_fn(x["a"], x["w"])[0] + bf(acc_fn(x["ta"], x["tw"])[0]))
    else:
        acc_t = acc_fn(*gb.with_tail(x["a"], x["w"], x["ta"], x["tw"]), **kw)[0]
    acc_g = acc_fn(x["a"], x["w_gelu"])[0]
    b = x["bias"]
    y = f32(bf(acc) + b) if defect == "bias_after_bf16_acc" else f32(acc + b)
    y_t = f32(acc_t + b)
    y_g = f32(acc_g + b)
    gate = bf(x["gate"]) if defect == "gate_bf16" else x["gate"]
    res = bf(x["res"]) if defect == "residual_bf16" else x["res"]
    yb = bf(y) if defect == "branch_bf16" else y
    o = fma(gate, yb, res)
    o_t = fma(gate, bf(y_t) if defect == "branch_bf16" else y_t, res)
    ax = bf(o) if defect == "aux_scale_after_bf16" else o
    g = f32(gb.gelu64(y_g)[0])
    dgl = f32(acc_g * f32(gb.gelu64(x["pre"])[1]))
    return {
        "bias": store(y), "gelu": store(g), "gelu_aux.aux": store(y_g), "mul_dgelu": store(dgl),
        "lora.bias": store(y_t), "lora.f32_residual": o_t,
        "f32_residual": o, "aux_scale": store(f32(ax * x["scale"])), "aux_branch": store(f32(y * x["scale"])),
        "bf16_residual": store(fma(gate, yb, bf(x["res"]))),
        "row_stats": row_stats_emul(o, BN, from_bf16=defect == "row_stats_bf16", wrong_part=defect == "row_stats_wrong_part",
                                    no_zero=defect == "row_stats_unzeroed"),
    }


def reference_fwd(x):
    """{family: (ref, slack, fp32 output, ulps of the final rounding, tiny)} for emulate_fwd's outputs, from gemm_bounds."""
    acc, s, _ = gb.accumulate(x["a"], x["w"])
    acc_t, s_t, _ = gb.accumulate(*gb.with_tail(x["a"], x["w"], x["ta"], x["tw"]))
    acc_g, s_g, _ = gb.accumulate(x["a"], x["w_gelu"])
    y, sy = gb.bias_out(acc, s, x["bias"])
    y_t, sy_t = gb.bias_out(acc_t, s_t, x["bias"])
    y_g, sy_g = gb.bias_out(acc_g, s_g, x["bias"])
    o, so = gb.residual_out(y, sy, x["gate"], x["res"])
    o_t, so_t = gb.residual_out(y_t, sy_t, x["gate"], x["res"])
    ob, sob = gb.residual_out(y, sy, x["gate"], bf(x["res"]), bf16=True)
    ax, sax = gb.aux_out(o, gb.f32_total(o, so), x["scale"])
    axb, saxb = gb.aux_out(y, gb.f32_total(y, sy), x["scale"])
    return {
        "bias": (y, sy, False, 0.5, 0.0), "gelu": (*gb.gelu_out(y_g, sy_g), False, 1.0, gb.GELU_TINY),
        "gelu_aux.aux": (y_g, sy_g, False, 0.5, 0.0), "mul_dgelu": (*gb.dgelu_out(acc_g, s_g, x["pre"]), False, 0.5, 0.0),
        "lora.bias": (y_t, sy_t, False, 0.5, 0.0), "lora.f32_residual": (o_t, so_t, True, 0.5, 0.0),
        "f32_residual": (o, so, True, 0.5, 0.0), "aux_scale": (ax, sax, False, 0.5, 0.0),
        "aux_branch": (axb, saxb, False, 0.5, 0.0), "bf16_residual": (ob, sob, False, 0.5, 0.0),
    }


def check_row_stats(got, out_kernel, bn=BN):
    """Tally of row_stats_out against the kernel's own fp32 out, and whether the unused parts are exactly zero."""
    ref, slack, parts = gb.row_stats_ref(out_kernel, bn)
    t = gb.Tally("row_stats", fp32=True).add(got[:, :parts], ref, slack)
    zero = bool((got[:, parts:] == 0).all())
    return t, zero


def tallies(outs, refs):
    ts = {}
    for name, (ref, slack, fp32, c, tiny) in refs.items():
        ts[name] = gb.Tally(name, fp32=fp32, c=c, tiny=tiny).add(outs[name], ref, slack)
    return ts


def normwise_accepts(outs, refs):
    """Whether every family passes the suite's normwise checks: rel_err < 2e-4 for fp32 outputs, < 4e-3 for bf16 ones."""
    for name, (ref, _, fp32, _, _) in refs.items():
        rel = ((outs[name] - ref).norm() / ref.norm()).item()
        if rel >= (2e-4 if fp32 else 4e-3):
            return False
    return True


# ------------------------------------------------------------------------------------------------- split-K and conv
KT, MW, NW, SPLITS = 512, 64, 96, 3


def wgrad_inputs():
    a_t, w_t = bf(randn(KT, MW, seed=20)), bf(randn(KT, NW, seed=21))
    bucket = f32(randn(MW, NW, seed=22, scale=KT ** 0.5))
    return a_t, w_t, bucket


def emulate_wgrad(model, defect=None):
    a_t, w_t, bucket = wgrad_inputs()
    parts = MODELS[model](a_t.T.contiguous(), w_t.T.contiguous(), k_splits=SPLITS)
    out = bucket
    for p in reversed(parts):                       # arrival order is unknown: the last split first
        out = f32(out + (bf(p) if defect == "splitk_partials_bf16" else p))
    return out


def reference_wgrad():
    a_t, w_t, bucket = wgrad_inputs()
    acc, s, parts = gb.accumulate(a_t.T.contiguous(), w_t.T.contiguous(), k_splits=SPLITS)
    return bucket + acc, s + SPLITS * gb.U * (bucket.abs() + parts)


CB, CH, CW, CIN, COUT = 2, 6, 5, 64, 32


def conv_inputs():
    x = bf(randn(CB, CH, CW, CIN, seed=30))
    w = bf(randn(COUT, 3, 3, CIN, seed=31, scale=(9 * CIN) ** -0.5))
    bias, res = bf(randn(COUT, seed=32, scale=0.1)), bf(randn(CB * CH * CW, COUT, seed=33))
    return x, w, bias, res


def emulate_conv(model, defect=None):
    x, w, bias, res = conv_inputs()
    a = gb.im2col(x, 0, CB * CH * CW)
    acc = MODELS[model](a, w.reshape(COUT, -1))[0]
    store = bf_rz if defect == "rz_store" else bf
    y = f32(acc + bias)
    return store(y), store(fma(torch.ones_like(y), bf(y) if defect == "branch_bf16" else y, res))


def reference_conv():
    x, w, bias, res = conv_inputs()
    acc, s = gb.conv_accumulate(x, w)
    y, sy = gb.bias_out(acc, s, bias)
    o, so = gb.residual_out(y, sy, torch.ones_like(y), res, bf16=True)
    return (y, sy), (o, so)


# ------------------------------------------------------------------------------------------------- tests
@pytest.fixture(scope="module")
def fwd():
    x = fwd_inputs()
    return x, reference_fwd(x)


@pytest.mark.parametrize("model", ["seq", "trunc"])
def test_models_inside_every_bound(model, fwd):
    x, refs = fwd
    outs = emulate_fwd(x, model)
    for t in tallies(outs, refs).values():
        t.check()
    t, zero = check_row_stats(outs["row_stats"], outs["f32_residual"])
    t.check()
    assert zero, "row_stats_out: unused parts not zero"
    ref, slack = reference_wgrad()
    gb.Tally(f"wgrad split-K {SPLITS}", fp32=True).add(emulate_wgrad(model), ref, slack).check()
    (y, sy), (o, so) = reference_conv()
    cy, co = emulate_conv(model)
    gb.Tally("conv3x3", tiny=0).add(cy, y, sy).check()
    gb.Tally("conv3x3 residual").add(co, o, so).check()


FWD_DEFECTS = ["rz_store", "branch_bf16", "gate_bf16", "residual_bf16", "bias_after_bf16_acc", "lora_tail_own_acc_bf16",
               "acc_bf16_between_kblocks", "aux_scale_after_bf16", "row_stats_bf16", "row_stats_wrong_part",
               "row_stats_unzeroed"]


@pytest.mark.parametrize("defect", FWD_DEFECTS)
def test_forward_defect_rejected(defect, fwd):
    x, refs = fwd
    outs = emulate_fwd(x, "seq", defect)
    ts = tallies(outs, refs)
    rs, zero = check_row_stats(outs["row_stats"], outs["f32_residual"])
    failed = [n for n, t in ts.items() if not t.ok()] + ([] if rs.ok() else ["row_stats"]) + ([] if zero else ["row_stats zero parts"])
    old = normwise_accepts(outs, refs)             # no normwise check reads row_stats_out itself
    worst = {n: f"{t.worst:.2f}/{t.bias:+.3f}" for n, t in ts.items() if not t.ok()}
    print(f"{defect}: rejected by {failed} (max err/bound / bias {worst}); old normwise checks "
          f"{'ACCEPT' if old else 'reject'} it")
    assert failed, f"{defect} passes every bound"


@pytest.mark.parametrize("defect", ["rz_store", "branch_bf16"])
def test_conv_defect_rejected(defect):
    (y, sy), (o, so) = reference_conv()
    cy, co = emulate_conv("seq", defect)
    ty, to = gb.Tally("conv3x3").add(cy, y, sy), gb.Tally("conv3x3 residual").add(co, o, so)
    old = ((cy - y).norm() / y.norm()).item() < 4e-3 and ((co - o).norm() / o.norm()).item() < 4e-3
    print(f"conv {defect}: bias {ty.bias:+.3f} / {to.bias:+.3f}, max err/bound {ty.worst:.2f} / {to.worst:.2f}; "
          f"old normwise checks {'ACCEPT' if old else 'reject'} it")
    assert not (ty.ok() and to.ok())


def test_splitk_partials_bf16_rejected():
    ref, slack = reference_wgrad()
    got = emulate_wgrad("seq", "splitk_partials_bf16")
    t = gb.Tally("wgrad, bf16 partials", fp32=True).add(got, ref, slack)
    rel = ((got - ref).norm() / ref.norm()).item()
    print(f"splitk_partials_bf16: max err/bound {t.worst:.1f}; old normwise (2e-4) {'ACCEPT' if rel < 2e-4 else 'reject'}s it "
          f"(rel_err {rel:.2e})")
    assert not t.ok()


def test_bias_threshold_separates(fwd):
    """The models' bias statistics and the truncating store's, side by side: MAX_BIAS must sit between them."""
    x, refs = fwd
    model_bias = max(abs(t.bias) for m in MODELS for t in tallies(emulate_fwd(x, m), refs).values())
    rz = tallies(emulate_fwd(x, "seq", "rz_store"), refs)
    stored = [n for n in rz if not refs[n][2]]                  # the bf16 families
    rz_bias = min(abs(rz[n].bias) for n in stored)
    print(f"largest |bias| of the models {model_bias:.4f}; smallest |bias| of a truncating bf16 store {rz_bias:.4f}; "
          f"MAX_BIAS {gb.MAX_BIAS}")
    assert model_bias * 3 <= gb.MAX_BIAS <= rz_bias / 2.5


def test_accumulate_matches_direct_sum():
    """accumulate(): acc is the float64 product, the slack is 2^-23 (sum over steps of |prefix| + sum |a w|), computed
    directly here step by step, and splits restart the prefix."""
    a, w = bf(randn(5, 200, seed=40)), bf(randn(7, 200, seed=41))
    acc, s, parts = gb.accumulate(a, w, k_splits=2, budget=5 * 7 * 8 * 16 * 2)     # two row chunks
    torch.testing.assert_close(acc, a @ w.T, rtol=1e-13, atol=1e-13)
    ap, wp = gb.pad_k(a), gb.pad_k(w)
    want = torch.zeros(5, 7, dtype=F64)
    pa = torch.zeros(5, 7, dtype=F64)
    for lo, hi in gb.mn_splits(4, 2):
        P = torch.zeros(5, 7, dtype=F64)
        for st in range(lo * 4, hi * 4):
            k = slice(16 * st, 16 * st + 16)
            want += gb.U_ACC * (P.abs() + ap[:, k].abs() @ wp[:, k].abs().T)
            P = P + ap[:, k] @ wp[:, k].T
        pa += P.abs()
    torch.testing.assert_close(s, want, rtol=1e-12, atol=0)
    torch.testing.assert_close(parts, pa, rtol=1e-12, atol=0)
