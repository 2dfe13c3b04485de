"""GPU tests (-m gpu) of the optimizer kernels element by element against the float64 one-step references of optim_bounds.py:
the CAME step (optim.FlatCAME, pxa_came_flat), AdamW (lib.adamw_flat / optim.FlatAdamW, pxa_adamw_flat) and gradient
clipping (lib.grad_clip_flat, pxa_grad_clip_flat).

Every case writes a state through the flat state tensors (FlatCAME._views, the AdamW state buffers): a mature one
(optim_bounds.mature_came_state / mature_adamw_state, weights at init scale so that the update spans thousands of ulps) or the
zero state of step 1, takes ONE step and checks every output against the reference of that step from the exact fp32 state the
kernel started from.  The CAME shapes cover every tile-geometry edge of came_geom: 1-D lengths around the 2048-element tile,
kind-1 matrices (at most 4 x 4) with lead around the 256-matrix tile and the patch embedding's 1152 x 4 x 2 x 2, the 4 x 5 /
5 x 4 boundary to kind 2, kind-2 R, C around the 128 x 128 tile and the XL/2 linear shapes, all at unaligned bucket offsets.
Gradient edges: an unused parameter (zero gradient; FlatCAME steps it with momentum), a zero row, a zero column and a row of
1e-20 gradients (subnormal squares) inside kind-1 and kind-2 matrices, gradients spanning 2^-20 .. 2^20.  Clipping is checked
twice over: the norm against float64, and every clipped gradient at the ulp level against (g grad_scale) coef with coef
formed in fp32 from the kernel's own norm.

With -s every output prints its largest error / bound and both bias statistics."""
import time

import pytest
import torch

import optim_bounds as ob

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
    from pixart_sigma_b200.optim import FlatAdamW, FlatCAME
    from pixart_sigma_b200.parallel import GradBucketReducer


class _Params(torch.nn.Module):
    def __init__(self, shapes):
        super().__init__()
        self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.zeros(s)) for s in shapes])


def _edit_grad(kind, shape, g, gen):
    """A gradient edge on the fp32 CPU gradient g of a parameter of `shape`:
      "edges": matrices get a zero row (1), a zero column (2) and a row of ~1e-20 gradients (0) whose squares are fp32
               subnormals; 1-D parameters get a quarter of their gradients scaled down to ~1e-20;
      "wide":  magnitudes 1e-3 x 2^-20 .. 2^20 with random signs;
      "zero":  an unused parameter."""
    if kind == "zero":
        return torch.zeros_like(g)
    if kind == "wide":
        e = torch.randint(-20, 21, g.shape, generator=gen, dtype=torch.int32)
        mant = torch.randn(g.shape, generator=gen).sign() * (1 + torch.rand(g.shape, generator=gen))
        return 1e-3 * torch.ldexp(mant, e)
    g = g.clone()
    if len(shape) >= 2:
        assert shape[-2] >= 3 and shape[-1] >= 3
        g[..., 0, :] = 1e-20 * torch.randn(g[..., 0, :].shape, generator=gen)
        g[..., 1, :] = 0
        g[..., :, 2] = 0
    else:
        g[: g.numel() // 4] *= 1e-17
    return g


def run_came(shapes, *, steps=(1,), lrs=(2e-5,), wd=0.0, p_scale=0.02, zero=False, grads=None, seed=0, tag=""):
    """Build a FlatCAME over parameters of `shapes` (one bucket, after a 3-element bias that misaligns every offset), write a
    state (grads: per shape None or a gradient edge of `_edit_grad`), then per lr in `lrs` one step checked against the
    reference from the state read back before it."""
    model = _Params([(3,)] + list(shapes)).cuda()
    red = GradBucketReducer(model)
    opt = FlatCAME(red, lr=lrs[0], weight_decay=wd)
    assert sum(e["offset"] % 4 != 0 for e in opt.entries) >= len(shapes) // 2
    gen = torch.Generator().manual_seed(seed + 100)
    params = list(model.parameters())
    kinds = [None] + list(grads or [None] * len(shapes))
    with torch.no_grad():
        for k, (e, p) in enumerate(zip(opt.entries, params)):
            pv, g, m, st = ob.mature_came_state(tuple(p.shape), seed + k, p_scale=p_scale, zero=zero)
            if kinds[k]:
                g = _edit_grad(kinds[k], tuple(p.shape), g, gen)
            p.copy_(pv)
            p.grad.copy_(g)
            views = opt._views(e, p)
            views["exp_avg"].copy_(m)
            for name, v in st.items():
                views[name].copy_(v)
    for kind, p in zip(kinds, params):
        if kind == "edges" and p.dim() >= 2:
            g = p.grad
            assert not g[..., 1, :].any() and not g[..., :, 2].any() and g[..., 3:, 3:].abs().min() > 0
            tiny = g[..., 0, :].abs()
            assert tiny.max() < 1e-18 and (tiny.square() < 1.1754944e-38).all() and tiny.count_nonzero() > tiny.numel() // 2
        elif kind == "zero":
            assert not p.grad.any()
    tallies = {}
    opt.step_count = steps[0] - 1
    for lr in lrs:
        opt.lr = lr
        before = []
        for e, p in zip(opt.entries, params):
            views = opt._views(e, p)
            before.append((p.detach().double(), p.grad.double(), views["exp_avg"].double(),
                           {k: v.double() for k, v in views.items() if k != "exp_avg"}))
        opt.step()
        torch.cuda.synchronize()
        for ei, ((p0, g, m, st), e, p) in enumerate(zip(before, opt.entries, params)):
            ref = ob.came_reference(p0, g, m, st, lr=ob.f32(lr), weight_decay=wd)
            views = opt._views(e, p)
            got = {"param": p.detach(), "RMS": opt.rms[ei], **views}
            for k, r in ref.items():
                tallies.setdefault(k, ob.Tally(f"came {tag} {k}")).add(got[k], *r)
        # the next step reads whatever this one wrote: a new gradient, same scales
        with torch.no_grad():
            for p in params:
                p.grad.mul_(-0.5)
    for t in tallies.values():
        t.check()
    return opt


VEC = [(1,), (3,), (2047,), (2048,), (2049,), (5000,)]
SMALL = [(lead, r, c) for r, c in [(1, 1), (2, 3), (4, 4)] for lead in (1, 255, 256, 257, 4608)] + [(1152, 4, 2, 2)]
BOUNDARY = [(4, 5), (5, 4)]
KIND2 = [(2, r, c) for r in (1, 127, 128, 129, 257) for c in (1, 127, 128, 129, 257) if r > 4 or c > 4] + [(6, 3, 5, 7)]
XL = [(1152, 1152), (4608, 1152), (1152, 4608), (6912, 1152)]
SHAPES = {"vec": VEC, "small": SMALL, "boundary": BOUNDARY, "kind2": KIND2}


@pytest.mark.parametrize("group", list(SHAPES))
@pytest.mark.parametrize("state", ["mature", "mature-wd", "zero", "p~1"])
def test_came_step_matches_float64(group, state):
    t0 = time.perf_counter()
    kw = {"mature": {}, "mature-wd": {"wd": 3e-2}, "zero": {"zero": True}, "p~1": {"p_scale": 1.0, "lrs": (1e-4,)}}[state]
    run_came(SHAPES[group], steps=(1000,), tag=f"{group} {state}", **{"lrs": (2e-5, 7e-5), **kw})
    print(f"[optim] came {group} {state}: {time.perf_counter() - t0:.1f} s")


EDGES = [((300, 200), "edges"), ((5000,), "edges"), ((37, 4, 4), "edges"), ((9, 11), "zero"), ((129, 257), "edges"),
         ((64, 96), "wide"), ((3000,), "wide"), ((20, 3, 4), "wide")]


@pytest.mark.parametrize("step", [1, 10, 3000, 100000])
def test_came_step_with_gradient_edges(step):
    """The zero row / zero column / 1e-20 row edges on kind-1 and kind-2 matrices, 2^+-20 gradients on others, an unused
    parameter.  Step counts do not enter CAME (no bias correction), so each count draws its own states and gradients."""
    shapes, kinds = zip(*EDGES)
    assert {ob.came_geom(s)[0] for s, k in EDGES if k == "edges" and len(s) >= 2} == {1, 2}
    run_came(shapes, steps=(step,), lrs=(2e-5, 1e-4), wd=3e-2, grads=kinds, seed=step, tag=f"edges step {step}")


def test_came_step_on_the_xl_shapes():
    t0 = time.perf_counter()
    run_came(XL + [(1152,)], lrs=(2e-5,), tag="xl")
    print(f"[optim] came xl: {time.perf_counter() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------------------------ AdamW
@pytest.mark.parametrize("step", [1, 10, 1000, 3000, 100000])
@pytest.mark.parametrize("wd,eps,gs", [(3e-2, 1e-10, 1.0), (0.0, 1e-8, 2.0 ** -16), (3e-2, 1e-8, 2.0 ** -16), (0.0, 1e-10, 1.0)])
def test_adamw_step_matches_float64(step, wd, eps, gs):
    for n, zero in [(4, False), (40000, False), (1 << 20, step == 1), (1048580, False)]:
        p, g, m, v = (t.cuda() for t in ob.mature_adamw_state(n, step + n, zero=zero, g_scale=1e-3 / gs))
        ref = ob.adamw_reference(p.double(), g.double(), m.double(), v.double(), step=step, lr=1e-4, eps=eps, weight_decay=wd,
                                 grad_scale=gs)
        shadow = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        lib.adamw_flat(p, g, m, v, step=step, lr=1e-4, betas=(0.9, 0.999), eps=eps, weight_decay=wd, grad_scale=gs, shadow=shadow)
        torch.cuda.synchronize()
        got = {"param": p, "exp_avg": m, "exp_avg_sq": v}
        for k, r in ref.items():
            ob.Tally(f"adamw n={n} step {step} wd={wd} eps={eps} gs={gs}{' zero' if zero else ''} {k}").add(got[k], *r).check()
        assert torch.equal(shadow, p.to(torch.bfloat16))


def test_flat_adamw_leaves_bucket_padding_and_steps_every_parameter():
    """FlatAdamW over buckets whose lengths are padded to a multiple of 4: the padding stays 0, every parameter matches."""
    model = _Params([(3,), (37, 53), (5,), (9, 11), (2,)]).cuda()
    red = GradBucketReducer(model)
    opt = FlatAdamW(red, lr=1e-4, eps=1e-10, weight_decay=3e-2)
    assert red.buckets[0]["flat"].numel() > sum(p.numel() for p in model.parameters())
    n = sum(p.numel() for p in model.parameters())
    p0, g, m, v = ob.mature_adamw_state(n, 9)
    with torch.no_grad():
        red.buckets[0]["flat_param"][:n].copy_(p0)
        red.buckets[0]["flat"][:n].copy_(g)
        opt.state[0]["exp_avg"][:n].copy_(m)
        opt.state[0]["exp_avg_sq"][:n].copy_(v)
    opt.step_count = 2999
    opt.step()
    torch.cuda.synchronize()
    ref = ob.adamw_reference(p0.double(), g.double(), m.double(), v.double(), step=3000, lr=1e-4, eps=1e-10, weight_decay=3e-2)
    got = {"param": red.buckets[0]["flat_param"][:n], "exp_avg": opt.state[0]["exp_avg"][:n],
           "exp_avg_sq": opt.state[0]["exp_avg_sq"][:n]}
    for k, r in ref.items():
        ob.Tally(f"FlatAdamW {k}").add(got[k].cpu(), *r).check()
    for t in (red.buckets[0]["flat_param"], opt.state[0]["exp_avg"], opt.state[0]["exp_avg_sq"]):
        assert not t[n:].any()


# ------------------------------------------------------------------------------------------------------------------ clip
def _check_clip(grads, lengths, max_norm, gs, tag):
    """Clip `grads` in place and check the norm against float64 and every clipped gradient against (g gs) coef, coef formed
    from the kernel's norm; float64 copies are made one bucket at a time."""
    before = [g.clone() for g in grads]
    partials = torch.empty(lib.GRAD_CLIP_PARTS, device="cuda")
    total = torch.empty((), device="cuda")
    lib.grad_clip_flat(grads, partials, total, max_norm=max_norm, grad_scale=gs, lengths=lengths)
    torch.cuda.synchronize()
    t_ref, t_slack = ob.clip_norm_reference(before, lengths, grad_scale=gs)
    one = lambda t: t.reshape(1)
    ob.Tally(f"clip {tag} norm").add(one(total), one(t_ref), one(t_slack), one(t_ref)).check()
    tal = ob.Tally(f"clip {tag} grads")
    for g, b, n in zip(grads, before, lengths):
        tal.add(g[:n], *ob.clip_bucket_reference(b, n, total.item(), max_norm=max_norm, grad_scale=gs))
        assert torch.equal(g[n:], b[n:])                           # padding untouched
    tal.check()
    return t_ref.item()


@pytest.mark.parametrize("max_norm", [0.01, 1e4])
@pytest.mark.parametrize("gs", [1.0, 2.0 ** -16])
def test_clip_matches_float64(max_norm, gs):
    gen = torch.Generator().manual_seed(3)
    lengths = [1, 6, 4099, 1200003, 3 * (1 << 20) + 2]
    grads = [((0.01 / gs) * torch.randn(n + 3, generator=gen)).cuda() for n in lengths]
    norm = _check_clip(grads, lengths, max_norm, gs, f"max_norm={max_norm} gs={gs}")
    assert (norm > max_norm) == (max_norm == 0.01)


def test_clip_on_the_xl_bucket_set():
    """The 29 gradient buckets of PixArtMS-XL/2 (610.9 M gradients) against the float64 norm, clipped element by element."""
    from pixart_sigma_b200 import PixArtMS_XL_2
    t0 = time.perf_counter()
    with torch.device("cuda"):
        model = PixArtMS_XL_2(input_size=128)
    red = GradBucketReducer(model)
    torch.manual_seed(11)
    for p in model.parameters():
        p.grad.normal_().mul_(1e-3)
    grads = [b["flat"] for b in red.buckets]
    lengths = [sum(p.numel() for p in b["params"]) for b in red.buckets]
    assert len(grads) == 29
    torch.cuda.reset_peak_memory_stats()
    _check_clip(grads, lengths, 0.01, 1.0, "xl")
    print(f"[optim] clip xl: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
