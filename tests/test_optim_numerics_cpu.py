"""CPU checks of the optimizer bounds in optim_bounds.py against a float32 emulation of the kernels (pxa_came_flat,
pxa_adamw_flat, pxa_grad_clip_flat) that follows their operation order: the per-lane / per-warp / per-tile partial sums and
their fixed-order reductions, fmaf where the kernels call it, one fp32 rounding per operation elsewhere.  They show that
- the correct emulation stays inside every bound, from mature states and from the zero state, with both bias statistics
  within optim_bounds.MAX_BIAS (over MIN_BIAS_N elements or more).  An output whose only error is its final rounding (a 1-D
  parameter without weight decay, say) reaches err / bound ~ 1: the bound's last term is the half ulp a correctly rounded
  result may be off;
- the bounds reject defects of the size of the rounding: the parameter (CAME, AdamW), exp_avg (AdamW) or clipped gradients
  written with round-toward-zero, AdamW's fp32 (1 - beta) and bias corrections of the fp32 betas (the pre-fix
  pxa_adamw_flat), CAME's omb formed in fp32, the second-moment and instability row means taken before the statistics'
  update, the clip divisor taken from one tile's sum;
- the normwise checks of test_came_gpu.py (1e-5 per tensor against the fp32 oracle, 5 steps from zero) and
  test_flat_adamw_matches_torch_adamw (1e-6 on the parameters, 3 steps from zero) accept the round-toward-zero writes and
  the pre-fix AdamW.  (CAME's fp32 omb moves exp_avg_res_col 1.7e-4 at step 1 and a stale row mean zeroes it, so those two
  only escape them from a mature state.)
CAME's exp_avg written toward zero is not rejected: its bound carries rsqrtf's 2 ulps through u, ~6 ulps of exp_avg, and the
truncation moves its bias by only -0.03.

With -s every case prints its largest error / bound and biases.
"""
import math

import pytest
import torch

import optim_bounds as ob
from oracle import came_oracle as co

F = torch.float32


def _f(x):
    return torch.as_tensor(x, dtype=F)


def fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def rsqrt(x):
    return x.double().rsqrt().float()


def rz(x64):
    """float64 -> fp32 rounded toward zero."""
    y = x64.float()
    over = y.double().abs() > x64.abs()
    return torch.where(over, torch.nextafter(y, torch.zeros_like(y)), y)


def seq(x, dim):
    """fp32 sum along dim, one term after the other, from 0."""
    x = x.movedim(dim, -1)
    acc = torch.zeros(x.shape[:-1], dtype=F)
    for k in range(x.shape[-1]):
        acc = acc + x[..., k]
    return acc


def sq_chain(x, dim):
    """acc = fmaf(x, x, acc) along dim, from 0."""
    x = x.movedim(dim, -1)
    acc = torch.zeros(x.shape[:-1], dtype=F)
    for k in range(x.shape[-1]):
        acc = fma(x[..., k], x[..., k], acc)
    return acc


def tree32(x):
    """The xor-shuffle tree over the last dim (32 lanes)."""
    for o in (16, 8, 4, 2, 1):
        x = x[..., :o] + x[..., o:2 * o]
    return x[..., 0]


def block_sum(x):
    """block_sum of optim_sm90.cu over the last dim (256 threads): a shuffle tree per warp, then the warps in order."""
    return seq(tree32(x.reshape(*x.shape[:-1], ob.WARPS, 32)), -1)


def strided_then_block(x):
    """Thread i sums elements i, i + 256, ... in order, then block_sum (clip_divisor, the finalisation's row mean)."""
    n = x.shape[-1]
    k = max(-(-n // ob.THREADS), 1)
    xp = torch.zeros(*x.shape[:-1], k * ob.THREADS, dtype=F)
    xp[..., :n] = x
    return block_sum(seq(xp.reshape(*x.shape[:-1], k, ob.THREADS), -2))


def _pad(x, *sizes):
    out = torch.zeros(*sizes, dtype=F)
    out[tuple(slice(0, s) for s in x.shape)] = x
    return out


class CameEmu:
    """One parameter's pxa_came_flat step in fp32, phase by phase as the kernels run it."""

    def __init__(self, shape, lr, eps, clip, betas, wd, defect=None):
        self.kind, self.lead, self.R, self.C, self.tiles = ob.came_geom(tuple(shape))
        self.shape, self.lr, self.defect = shape, _f(lr), defect
        self.b = [_f(ob.f32(b)) for b in betas]
        self.omb = [(_f(1.0) - self.b[i]) if defect == "omb_f32" else _f(ob.f32(1.0 - b)) for i, b in enumerate(betas)]
        self.eps1, self.eps2, self.clip, self.wd = _f(eps[0]), _f(eps[1]), _f(clip), _f(wd)

    # sums of a (lead, R, C) array as the kernels form them
    def row_sums(self, x):
        if self.kind == 1:
            return seq(x, -1)
        CT = -(-self.C // ob.TC)
        xp = _pad(x, self.lead, self.R, CT * ob.TC).reshape(self.lead, self.R, CT, 4, 32)
        return seq(tree32(seq(xp, -2)), -1)

    def col_sums(self, x):
        if self.kind == 1:
            return seq(x, -2)
        RT = -(-self.R // ob.TR)
        xp = _pad(x, self.lead, RT * ob.TR, self.C).reshape(self.lead, RT, ob.TR // ob.WARPS, ob.WARPS, self.C)
        return seq(seq(seq(xp, 2), 2), 1)

    def row_mean(self, row):
        return (seq(row, -1) if self.kind == 1 else strided_then_block(row)) / _f(self.R)

    def tile_sq_sums(self, x):
        """Per-tile sums of x^2 in tile order (phase 0 / 1 / 3)."""
        if self.kind == 0:
            xp = _pad(x.reshape(-1), self.tiles * ob.VEC_TILE).reshape(self.tiles, ob.VEC_TILE // ob.THREADS, ob.THREADS)
            return block_sum(sq_chain(xp, 1))
        if self.kind == 1:
            xp = _pad(x.reshape(self.lead, -1), self.tiles * ob.SMALL_TILE, self.R * self.C)
            return block_sum(sq_chain(xp.reshape(self.tiles, ob.SMALL_TILE, -1), -1))
        RT, CT = -(-self.R // ob.TR), -(-self.C // ob.TC)
        xp = _pad(x, self.lead, RT * ob.TR, CT * ob.TC).reshape(self.lead, RT, ob.TR // ob.WARPS, ob.WARPS, CT, 4, 32)
        th = xp.permute(0, 1, 4, 3, 6, 2, 5).reshape(self.lead, RT, CT, ob.THREADS, -1)     # thread = warp * 32 + lane
        return block_sum(sq_chain(th, -1)).reshape(-1)

    def factors(self, row, col, rm):
        q = row / rm[..., None]
        return rsqrt(q)[..., :, None] * rsqrt(col)[..., None, :]

    def step(self, p, g, m, state):
        out = {}
        b1, b2, b3 = self.b
        o1, o2, o3 = self.omb
        x = g * g + self.eps1
        if self.kind == 0:
            v = state["exp_avg_sq"] * b2 + o2 * x
            out["exp_avg_sq"] = v
            f = rsqrt(v)
        else:
            L, R, C = self.lead, self.R, self.C
            x3 = x.reshape(L, R, C)
            row0, col0 = (state[k].reshape(L, -1) for k in ("exp_avg_sq_row", "exp_avg_sq_col"))
            row = row0 * b2 + o2 * (self.row_sums(x3) / _f(C))
            col = col0 * b2 + o2 * (self.col_sums(x3) / _f(R))
            out["exp_avg_sq_row"], out["exp_avg_sq_col"] = row, col
            rm = self.row_mean(row0 if self.defect == "stale_rm" else row)
            f = self.factors(row, col, rm).reshape(self.shape)
        u = f * g
        ts = self.tile_sq_sums(u.reshape(self.lead, self.R, self.C) if self.kind else u)
        s = ts[0] if self.defect == "clip_one_tile" else strided_then_block(ts)
        div = torch.clamp_min(torch.sqrt(s) / _f(math.sqrt(p.numel())) / self.clip, 1.0)
        uc = u / div
        mm = m * b1
        if self.defect == "exp_avg_rz":
            m1 = rz(mm.double() + (o1 * uc).double())
        else:
            m1 = mm + o1 * uc
        out["exp_avg"] = m1
        if self.kind == 0:
            upd = m1
        else:
            d = uc - m1
            r3 = (d * d + self.eps2).reshape(L, R, C)
            rrow0, rcol0 = (state[k].reshape(L, -1) for k in ("exp_avg_res_row", "exp_avg_res_col"))
            rrow = rrow0 * b3 + o3 * (self.row_sums(r3) / _f(C))
            rcol = rcol0 * b3 + o3 * (self.col_sums(r3) / _f(R))
            out["exp_avg_res_row"], out["exp_avg_res_col"] = rrow, rcol
            rm3 = self.row_mean(rrow0 if self.defect == "stale_rm" else rrow)
            upd = self.factors(rrow, rcol, rm3).reshape(self.shape) * m1
        q = p
        if float(self.wd) != 0.0:
            q = q + (-self.wd * self.lr) * q
        if self.defect == "param_rz":
            out["param"] = rz(q.double() - (upd * self.lr).double())
        else:
            out["param"] = q - upd * self.lr
        pts = self.tile_sq_sums(p.reshape(self.lead, self.R, self.C) if self.kind else p)
        k = -(-pts.numel() // 32)
        sp = tree32(seq(_pad(pts, k * 32).reshape(k, 32), 0))
        out["RMS"] = torch.sqrt(sp) / _f(math.sqrt(p.numel()))
        for key in [k for k in out if k.startswith("exp_avg_") and k != "exp_avg_sq"]:
            out[key] = out[key].reshape(state[key].shape)
        return out


def came_check(shape, seed, *, lr=2e-5, wd=0.0, p_scale=0.02, zero=False, defect=None, eps=(1e-30, 1e-16), clip=1.0,
               betas=(0.9, 0.999, 0.9999)):
    """One emulated CAME step from a (mature or zero) state against the float64 reference: {output: Tally}."""
    p, g, m, st = ob.mature_came_state(shape, seed, p_scale=p_scale, zero=zero)
    lr = ob.f32(lr)
    got = CameEmu(shape, lr, eps, clip, betas, wd, defect).step(p, g, m, st)
    ref = ob.came_reference(p.double(), g.double(), m.double(), {k: v.double() for k, v in st.items()}, lr=lr, eps=eps,
                            clip_threshold=clip, betas=betas, weight_decay=wd)
    tag = f"came {tuple(shape)} wd={wd} p~{p_scale}{' zero' if zero else ''}{' ' + defect if defect else ''}"
    return {k: ob.Tally(f"{tag} {k}").add(got[k], *ref[k]) for k in ref}


def adamw_emulate(p, g, m, v, *, step, lr, betas, eps, wd, gs, defect=None):
    """pxa_adamw_flat's arithmetic in fp32; defect "parent": the pre-fix kernel (fp32 hyper-parameters, 1.0f - beta in the
    kernel, bias corrections of the fp32 betas, decay 1.0f - lr * wd in fp32)."""
    b1, b2 = _f(ob.f32(betas[0])), _f(ob.f32(betas[1]))
    if defect == "parent":
        o1, o2 = _f(1.0) - b1, _f(1.0) - b2
        bc1, bc2 = 1.0 - float(b1) ** step, 1.0 - float(b2) ** step
        decay = _f(1.0) - _f(lr) * _f(wd)
    else:
        o1, o2 = _f(ob.f32(1.0 - betas[0])), _f(ob.f32(1.0 - betas[1]))
        bc1, bc2 = 1.0 - betas[0] ** step, 1.0 - betas[1] ** step
        decay = _f(1.0 - lr * wd)
    ss, isb = _f(lr / bc1), _f(1.0 / math.sqrt(bc2))
    gk = g * _f(gs)
    m1 = fma(b1.expand_as(m), m, o1 * gk)
    v1 = fma(b2.expand_as(v), v, o2 * gk * gk)
    den = torch.sqrt(v1) * isb + _f(eps)
    p1 = fma((-ss).expand_as(p), m1 / den, p * decay)
    if defect == "param_rz":
        p1 = rz((-ss).double() * (m1 / den).double() + (p * decay).double())
    if defect == "exp_avg_rz":
        m1 = rz(b1.double() * m.double() + (o1 * gk).double())
        p1 = fma((-ss).expand_as(p), m1 / den, p * decay)
    return {"param": p1, "exp_avg": m1, "exp_avg_sq": v1}


def adamw_check(n, seed, *, step, lr=1e-4, wd=3e-2, eps=1e-10, gs=1.0, zero=False, defect=None, p_scale=0.02):
    p, g, m, v = ob.mature_adamw_state(n, seed, zero=zero, p_scale=p_scale, g_scale=1e-3 / gs)
    kw = dict(step=step, lr=lr, betas=(0.9, 0.999), eps=eps)
    got = adamw_emulate(p, g, m, v, wd=wd, gs=gs, defect=defect, **kw)
    ref = ob.adamw_reference(p.double(), g.double(), m.double(), v.double(), weight_decay=wd, grad_scale=gs, **kw)
    tag = f"adamw step {step} wd={wd} eps={eps} gs={gs}{' zero' if zero else ''}{' ' + defect if defect else ''}"
    return {k: ob.Tally(f"{tag} {k}").add(got[k], *ref[k]) for k in ref}


def _check_all(tallies):
    for t in tallies.values():
        t.check()


CAME_SHAPES = [(5000,), (3,), (2049,), (300, 4, 2, 2), (70, 2, 3), (5, 4), (4, 5), (200, 300), (6, 3, 5, 7), (129, 257)]


@pytest.mark.parametrize("shape", CAME_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("wd,p_scale,zero", [(0.0, 0.02, False), (3e-2, 0.02, False), (0.0, 1.0, False), (0.0, 0.02, True)],
                         ids=["mature", "mature-wd", "p~1", "zero"])
def test_came_emulation_is_inside_the_bounds(shape, wd, p_scale, zero):
    _check_all(came_check(shape, 1, wd=wd, p_scale=p_scale, zero=zero, lr=1e-4 if p_scale == 1.0 else 2e-5))


@pytest.mark.parametrize("step", [1, 10, 1000, 3000, 100000])
@pytest.mark.parametrize("wd,eps,gs", [(3e-2, 1e-10, 1.0), (0.0, 1e-8, 2.0 ** -16)])
def test_adamw_emulation_is_inside_the_bounds(step, wd, eps, gs):
    _check_all(adamw_check(40000, step, step=step, wd=wd, eps=eps, gs=gs))
    if step == 1:
        _check_all(adamw_check(40000, 7, step=1, wd=wd, eps=eps, gs=gs, zero=True))


def _rejected(tallies):
    return [t.name for t in tallies.values() if not t.ok()]


@pytest.mark.parametrize("defect,shape,zero", [
    ("param_rz", (5000,), False), ("param_rz", (200, 300), False),
    ("omb_f32", (200, 300), True), ("omb_f32", (5000,), False), ("stale_rm", (200, 300), False),
    ("clip_one_tile", (300, 200), False), ("clip_one_tile", (5000,), False)])
def test_came_bounds_reject_defects(defect, shape, zero):
    tallies = came_check(shape, 2, defect=defect, zero=zero)
    for t in tallies.values():
        t.report()
    assert _rejected(tallies), f"{defect} passed every bound"


@pytest.mark.parametrize("step,zero", [(1, True), (10, False), (1000, False), (3000, False), (100000, False)])
def test_adamw_bounds_reject_the_pre_fix_kernel(step, zero):
    tallies = adamw_check(40000, 3, step=step, zero=zero, defect="parent")
    for t in tallies.values():
        t.report()
    assert _rejected(tallies), "the pre-fix pxa_adamw_flat passed every bound"


@pytest.mark.parametrize("defect,out", [("param_rz", "param"), ("exp_avg_rz", "exp_avg")])
def test_adamw_bounds_reject_truncated_writes(defect, out):
    tallies = adamw_check(40000, 4, step=1000, defect=defect)
    for t in tallies.values():
        t.report()
    assert f"{defect} {out}" in " ".join(_rejected(tallies))


# ------------------------------------------------------------------------------------ what the normwise checks accept
def _old_came_check(defect, steps=5, lr=1e-2, wd=0.0):
    """test_came_gpu's check: from the zero state, `steps` steps of the emulation (with `defect`) and of the fp32 oracle on
    randn weights and 0.1 randn gradients; the largest normwise relative error over every parameter and state tensor."""
    shapes = [(37, 53), (6, 3, 5, 7), (300, 4, 2, 2), (200, 300), (5000,)]
    gen = torch.Generator().manual_seed(0)
    worst = 0.0
    for shape in shapes:
        p0 = torch.randn(*shape, generator=gen)
        emu = CameEmu(shape, ob.f32(lr), (1e-30, 1e-16), 1.0, (0.9, 0.999, 0.9999), wd, defect)
        p, ref = p0.clone(), [p0.clone()]
        st = {k: v.float() for k, v in ob.mature_came_state(shape, 0, zero=True)[3].items()}
        m = torch.zeros(shape)
        states = [{}]
        for _ in range(steps):
            g = 0.1 * torch.randn(*shape, generator=gen)
            out = emu.step(p, g, m, st)
            p, m = out["param"], out["exp_avg"]
            st = {k: out[k] for k in st}
            co.came_step(ref, [g], states, lr=lr, weight_decay=wd)
        pairs = [(p, ref[0]), (m, states[0]["exp_avg"])] + [(st[k], states[0][k]) for k in st]
        worst = max(worst, max(((a.double() - b.double()).norm() / b.double().norm()).item() for a, b in pairs))
    return worst


@pytest.mark.parametrize("defect", ["param_rz"])
def test_old_came_normwise_check_accepts_rounding_sized_defects(defect):
    """test_came_gpu's bound (1e-5 per tensor, 5 steps from zero, against the fp32 oracle) passes the defect that
    test_came_bounds_reject_defects rejects; the correct emulation sits at the same level."""
    err, base = _old_came_check(defect), _old_came_check(None)
    print(f"old CAME normwise check: {defect} {err:.2e}, correct emulation {base:.2e}")
    assert err <= 1e-5


@pytest.mark.parametrize("defect", ["parent", "param_rz", "exp_avg_rz"])
def test_old_adamw_normwise_check_accepts_rounding_sized_defects(defect):
    """test_flat_adamw_matches_torch_adamw's check (three steps from zero on a 37 x 53 Linear, lr 2e-3, normwise 1e-6 on the
    parameters against torch.optim.AdamW) passes the pre-fix kernel's arithmetic and the truncated writes."""
    torch.manual_seed(0)
    lin = torch.nn.Linear(53, 37)
    params = [p.detach().clone().reshape(-1) for p in lin.parameters()]
    ref = [torch.nn.Parameter(p.clone()) for p in params]
    opt = torch.optim.AdamW(ref, lr=2e-3, eps=1e-10, weight_decay=3e-2)
    state = [(torch.zeros_like(p), torch.zeros_like(p)) for p in params]
    for s in range(1, 4):
        grads = [torch.randn(p.shape) for p in params]
        for q, g in zip(ref, grads):
            q.grad = g.clone()
        opt.step()
        for i, (p, g) in enumerate(zip(params, grads)):
            out = adamw_emulate(p, g, *state[i], step=s, lr=2e-3, betas=(0.9, 0.999), eps=1e-10, wd=3e-2, gs=1.0,
                                defect=defect)
            params[i], state[i] = out["param"], (out["exp_avg"], out["exp_avg_sq"])
    err = (torch.cat(params).double() - torch.cat([q.detach() for q in ref]).double()).norm() / torch.cat(
        [q.detach() for q in ref]).double().norm()
    print(f"old AdamW normwise check, {defect}: {err.item():.2e}")
    assert err <= 1e-6


# ------------------------------------------------------------------------------------ clipping
def clip_emulate(grads, lengths, max_norm, gs, defect=None):
    """pxa_grad_clip_flat in fp32: per-thread fmaf chains over the float4s and tails of every bucket, block_sum per CTA,
    4 partials per thread and block_sum; then (g gs) coef.  defect "rz": the clipped gradients written toward zero."""
    T = ob.CLIP_PARTS * ob.THREADS
    acc = torch.zeros(T, dtype=F)
    gs = _f(gs)
    for g, n in zip(grads, lengths):
        x = g[:n] * gs
        n4 = n // 4
        for c in range(-(-n4 // T)):
            blk = x[4 * c * T: 4 * min((c + 1) * T, n4)].reshape(-1, 4)
            for k in range(4):
                acc[:blk.shape[0]] = fma(blk[:, k], blk[:, k], acc[:blk.shape[0]])
        tail = x[4 * n4:]
        acc[:tail.numel()] = fma(tail, tail, acc[:tail.numel()])
    partials = block_sum(acc.reshape(ob.CLIP_PARTS, ob.THREADS))
    total = torch.sqrt(block_sum(seq(partials.reshape(ob.CLIP_PARTS // ob.THREADS, ob.THREADS), 0)))
    coef = torch.clamp_max(_f(max_norm) / (total + _f(1e-6)), 1.0)
    if defect == "rz":
        return total, [rz((g[:n] * gs).double() * coef.double()) for g, n in zip(grads, lengths)]
    return total, [(g[:n] * gs) * coef for g, n in zip(grads, lengths)]


def clip_check(max_norm, gs, defect=None):
    gen = torch.Generator().manual_seed(5)
    lengths = [1, 6, 4099, 1200003]
    grads = [(0.1 / gs) * torch.randn(n + 3, generator=gen) for n in lengths]
    total, out = clip_emulate(grads, lengths, max_norm, gs, defect)
    t_ref, t_slack = ob.clip_norm_reference(grads, lengths, grad_scale=gs)
    one = lambda t: t.reshape(1)
    norm = ob.Tally(f"clip max_norm={max_norm} gs={gs} norm").add(one(total), one(t_ref), one(t_slack), one(t_ref))
    tal = ob.Tally(f"clip max_norm={max_norm} gs={gs}{' ' + defect if defect else ''} grads")
    for o, g, n in zip(out, grads, lengths):
        tal.add(o, *ob.clip_bucket_reference(g, n, total, max_norm=max_norm, grad_scale=gs))
    return {"norm": norm, "grads": tal}


@pytest.mark.parametrize("max_norm,gs", [(0.01, 1.0), (1e4, 1.0), (0.05, 2.0 ** -16), (1e4, 2.0 ** -16)])
def test_clip_emulation_is_inside_the_bounds(max_norm, gs):
    _check_all(clip_check(max_norm, gs))


@pytest.mark.parametrize("gs", [1.0, 2.0 ** -16])
def test_clip_bounds_reject_a_truncated_write(gs):
    tallies = clip_check(0.01, gs, "rz")
    tallies["grads"].report()
    assert not tallies["grads"].ok()
