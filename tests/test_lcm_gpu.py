"""GPU tests (-m gpu) of the LCM kernels and drivers (pixart_sigma_b200/lcm.py) against fp64 formulas, the oracle
(oracle/lcm_oracle.py) and the reference fixtures (tests/golden/lcm_*.pt).  Each test prints its measured error (shown
with `pytest -rP` or `-s`).

Tolerances:
  * pxa_lcm_step vs its fp32 formula: 1e-6 (the kernel rounds each operation as the reference's torch operations do);
  * sampler loop with the toy denoiser vs the reference fixture: 1e-5;
  * sampler loop around a depth-2 PixArtMS vs the oracle loop on the same bf16-rounded weights: 2e-2 (bf16 GEMM operands);
  * teacher target vs fp64: 1e-6; loss vs fp64: 1e-6 relative; gradient vs fp64 autograd: 1e-5;
  * full distillation step vs the oracle (same bf16-rounded weights): loss 2e-3, gradients 2e-2 (L2) / 3e-2 (Huber: see the
    test), the bounds of test_training_gpu.py;
  * graphed step vs eager: 1e-4, the reorder tolerance of test_training_gpu.py (atomics in the backward reorder sums).
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dpm_oracle as do            # noqa: E402
from oracle import lcm_oracle as lo            # noqa: E402
from oracle import pixart_oracle as po         # noqa: E402
from oracle.gen_golden_lcm import SAMPLER_CASES  # noqa: E402
from oracle.gen_golden_train import train_inputs  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"

if torch.cuda.is_available():
    from pixart_sigma_b200 import build_model, lib
    from pixart_sigma_b200.graph import GraphedForward
    from pixart_sigma_b200.lcm import GraphedLCMStep, LCMDistiller, LCMSampler, LCMScheduler, distill_table
    from pixart_sigma_b200.optim import FlatCAME, clip_grad_norm_
    from pixart_sigma_b200.parallel import GradBucketReducer


def _log(line):
    print(line)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _gold(name):
    return torch.load(os.path.join(GOLD, name + ".pt"))


# ------------------------------------------------------------------------------------------------- sampler
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("form", ["multi", "last", "one"])
def test_step_kernel_matches_formula(dtype, form):
    g = torch.Generator().manual_seed(3)
    n, h, w = 3, 24, 20
    out = torch.randn(n, 8, h, w, generator=g).to(dtype).to(DEV)[:, :4]
    x, z = (torch.randn(n, 4, h, w, generator=g).to(DEV) for _ in range(2))
    sch = LCMScheduler()
    sch.set_timesteps(1 if form == "one" else 4, 50)
    i = {"multi": 1, "last": 3, "one": 0}[form]
    k = sch.step_scalars(i, sch.timesteps[i])
    if form == "one":
        z = torch.full_like(z, float("nan"))              # c_noise = 0: must not be read
        assert k["c_noise"] == 0.0
    eps = out.float()
    sa, sb, cs, co, cp, cn = (torch.tensor(k[n_], dtype=torch.float32, device=DEV)
                              for n_ in ("sqrt_alpha", "sqrt_beta", "c_skip", "c_out", "c_prev", "c_noise"))
    x0 = (x - sb * eps) / sa
    den = co * x0 + cs * x
    nxt = den if form == "one" else cp * den + cn * z
    gd, gn = torch.empty_like(x), torch.empty_like(x)
    lib.lcm_step(out, x, z if k["c_noise"] else None, gd, gn, **k)
    ed, en = _rel(gd, den), _rel(gn, nxt)
    _log(f"lcm_step {dtype} {form}: denoised rel {ed:.2e} (max abs {float((gd - den).abs().max()):.2e}), next rel {en:.2e}")
    assert ed < 1e-6 and en < 1e-6 and torch.isfinite(gn).all()


@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("name", sorted(SAMPLER_CASES))
def test_loop_with_toy_denoiser_matches_reference_fixture(name, graph):
    gd = _gold(name)
    steps = gd["case"]["steps"]
    sampler = LCMSampler(do.toy_model)
    kw = dict(cond=gd["cond"].to(DEV))
    draws = gd["draws"] if steps > 1 else None
    out = sampler.sample(gd["x_T"].to(DEV), steps=steps, model_kwargs=kw, noise=draws, cuda_graph=graph)
    err = _rel(out, gd["out"])
    if graph:                                             # a second replay of the same capture
        err = max(err, _rel(sampler.sample(gd["x_T"].to(DEV), steps=steps, model_kwargs=kw, noise=draws, cuda_graph=True),
                            gd["out"]))
    _log(f"lcm loop {name} graph={graph}: rel err vs reference {err:.2e}")
    assert err < 1e-5
    if not graph:                                         # drawing itself: the reference's CPU draws, generator state after
        torch.manual_seed(gd["seed"])
        out2 = sampler.sample(gd["x_T"].to(DEV), steps=steps, model_kwargs=kw)
        assert torch.equal(torch.get_rng_state(), gd["rng_after"])
        assert _rel(out2, gd["out"]) < 1e-5


def _model(cfg, sd, dtype=torch.bfloat16):
    kw = dict(type="PixArtMS", depth=cfg.depth, hidden_size=cfg.hidden_size, num_heads=cfg.num_heads, input_size=cfg.input_size,
              pe_interpolation=cfg.pe_interpolation, model_max_length=cfg.model_max_length)
    with torch.device(DEV):
        m = build_model(kw)
    m.load_state_dict(sd, strict=False)
    return m.to(dtype)


def _r(v):
    return v.to(torch.bfloat16).float()


def test_loop_around_pixartms_matches_oracle_loop():
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    sd = {k: _r(v) for k, v in po.synthetic_state_dict(cfg, seed=0).items()}
    m = _model(cfg, sd).eval()
    m.output_dtype = torch.float32
    x, _, y, mask = po.synthetic_inputs(cfg, 2, (32, 32), lens=[300, 77])
    torch.manual_seed(5)
    noise = LCMSampler.draw_noise(4, tuple(x.shape))
    got = LCMSampler(m).sample(x.to(DEV), steps=4, model_kwargs=dict(y=_r(y).to(DEV), mask=mask.to(DEV)), noise=noise)
    oracle = lambda xx, t, **kw: po.forward(sd, cfg, _r(xx), t.float(), _r(y), mask=mask)   # the kernels read bf16 x
    want, _ = lo.sample(oracle, x, steps=4, noise=noise)
    err = _rel(got, want)
    _log(f"lcm loop around PixArtMS depth 2 (4 steps): rel err vs oracle {err:.2e}")
    assert err < 2e-2


# ------------------------------------------------------------------------------------------------- distillation kernels
def _table_dev():
    rows = distill_table()[2]
    t = (lib.LcmRow * len(rows))(*[lib.LcmRow(**r) for r in rows])
    return rows, torch.frombuffer(bytearray(bytes(t)), dtype=torch.uint8).to(DEV)


def _f64_target(rows, index, teacher_out, x_t, w):
    b = x_t.shape[0]
    col = lambda k: torch.tensor([rows[int(i)][k] for i in index], dtype=torch.float64).view(b, 1, 1, 1).to(DEV)
    ec, eu = teacher_out[:b, :4].double(), teacher_out[b:, :4].double()
    xt = x_t.double()
    x0c, x0u = col("sra_s") * xt - col("srm1_s") * ec, col("sra_s") * xt - col("srm1_s") * eu
    return col("sqrt_acp") * (x0c + w * (x0c - x0u)) + col("sqrt_1macp") * (ec + w * (ec - eu)), col


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_teacher_target_and_consistency_loss_match_fp64(dtype):
    g = torch.Generator().manual_seed(8)
    b, h, w = 3, 16, 20
    rows, table = _table_dev()
    index = torch.tensor([0, 37, 49], dtype=torch.long, device=DEV)
    teacher_out = torch.randn(2 * b, 8, h, w, generator=g).to(dtype).to(DEV)
    x_t = torch.randn(b, 4, h, w, generator=g).to(DEV)
    x_prev = torch.empty_like(x_t)
    lib.lcm_teacher_target(teacher_out[:, :4], x_t, index, table, x_prev, w=4.5)
    want, col = _f64_target(rows, index.tolist(), teacher_out, x_t, 4.5)
    e_prev = _rel(x_prev, want)
    student = torch.randn(b, 8, h, w, generator=g).to(DEV)
    ema = (torch.randn(b, 8, h, w, generator=g) * 0.3).to(dtype).to(DEV)
    partials = torch.empty(lib.LCM_LOSS_PARTS, dtype=torch.float64, device=DEV)
    for loss_type, name in ((lib.LCM_HUBER, "huber"), (lib.LCM_L2, "l2")):
        runs = []
        for _ in range(2):
            d, loss = torch.empty_like(student), torch.empty((), device=DEV)
            lib.lcm_consistency_loss(student, ema[:, :4], x_t, x_prev, index, table, d, loss, partials, loss_type=loss_type,
                                     huber_c=1e-3)
            runs.append((loss.clone(), d.clone()))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])          # bitwise reproducible
        s64 = student.double().clone().requires_grad_(True)
        xt, xp = x_t.double(), x_prev.double()
        pred = col("cskip_s") * xt + col("cout_s") * (col("sra_s") * xt - col("srm1_s") * s64[:, :4])
        tgt = col("cskip_t") * xp + col("cout_t") * (col("sra_t") * xp - col("srm1_t") * ema[:, :4].double())
        dd = pred - tgt
        ref = torch.mean(torch.sqrt(dd ** 2 + 1e-6) - 1e-3) if name == "huber" else torch.mean(dd ** 2)
        ref.backward()
        e_loss = abs(float(runs[0][0]) - float(ref)) / abs(float(ref))
        e_grad = _rel(runs[0][1], s64.grad)
        sigma_zero = bool((runs[0][1][:, 4:] == 0).all())
        _log(f"lcm teacher/loss {dtype} {name}: x_prev rel {e_prev:.2e}, loss rel {e_loss:.2e}, grad rel {e_grad:.2e}, "
             f"sigma channels zero {sigma_zero}")
        assert e_loss < 1e-6 and e_grad < 1e-5 and sigma_zero
    assert e_prev < 1e-6


def _ema_table(entries):
    return torch.frombuffer(bytearray(bytes((lib.EmaBucket * len(entries))(*entries))), dtype=torch.uint8).to(DEV)


@pytest.mark.parametrize("which", ["xl2", "odd"])
def test_ema_flat_equals_reference_ema_update(which):
    if which == "xl2":
        with torch.device(DEV):
            model = build_model(dict(type="PixArtMS", depth=28, input_size=128, model_max_length=300))
    else:
        class Odd(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.blocks = torch.nn.ModuleList([torch.nn.Linear(37, 53), torch.nn.Linear(3, 1)])
                self.a = torch.nn.Parameter(torch.randn(7))
                self.b = torch.nn.Parameter(torch.randn(5, 3, 2))
        model = Odd().to(DEV)
    red = GradBucketReducer(model)
    red.flatten_params()
    g = torch.Generator(device=DEV).manual_seed(2)
    entries, masters, shadows, ref = [], [], [], []
    for bk in red.buckets:
        fp = bk["flat_param"]
        fp.copy_(torch.randn(fp.shape, device=DEV, generator=g))
        n = sum(p.numel() for p in bk["params"])
        m = torch.full_like(fp, 7.0)                                 # padding sentinel
        m[:n] = torch.randn(n, device=DEV, generator=g)
        sh = torch.full((fp.numel(),), -3.0, dtype=torch.bfloat16, device=DEV)
        masters.append(m)
        shadows.append(sh)
        ref.append([m[o:o + p.numel()].clone() for o, p in zip(_offsets(bk["params"]), bk["params"])])
        entries.append(lib.EmaBucket(master=m.data_ptr(), src=fp.data_ptr(), shadow=sh.data_ptr(), n=n))
    table = _ema_table(entries)
    args = dict(n_buckets=len(entries), max_n=max(e.n for e in entries), rate=0.95)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lib.ema_flat(table, **args)                              # no host sync
    finally:
        torch.cuda.set_sync_debug_mode("default")
    # reference: ema_update's d.mul_(rate).add_((1 - rate) * s) on the same fp32 tensors
    for bk, r in zip(red.buckets, ref):
        for d, p in zip(r, bk["params"]):
            d.mul_(0.95).add_((1 - 0.95) * p.data.reshape(-1))
    ok = True
    for bk, m, sh, r in zip(red.buckets, masters, shadows, ref):
        n = sum(p.numel() for p in bk["params"])
        ok &= torch.equal(m[:n], torch.cat(r)) and torch.equal(sh[:n], m[:n].to(torch.bfloat16))
        ok &= bool((m[n:] == 7.0).all()) and bool((sh[n:] == -3.0).all())
    # a graph replay is bitwise equal to an eager launch
    saved = [m.clone() for m in masters]
    lib.ema_flat(table, **args)
    eager = [m.clone() for m in masters]
    for m, s in zip(masters, saved):
        m.copy_(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lib.ema_flat(table, **args)
    for m, s in zip(masters, saved):
        m.copy_(s)
    graph.replay()
    same = all(torch.equal(m, e) for m, e in zip(masters, eager))
    _log(f"ema_flat {which}: {sum(e.n for e in entries)} parameters in {len(entries)} buckets, bitwise equal to ema_update "
         f"{ok}, graph replay equal {same}")
    assert ok and same


def _offsets(params):
    out, o = [], 0
    for p in params:
        out.append(o)
        o += p.numel()
    return out


# ------------------------------------------------------------------------------------------------- distiller
CFG = dict(depth=2, input_size=32, pe_interpolation=0.5)


def _distill_setup(loss_type="huber", checkpoint=False):
    cfg = po.OracleConfig(**CFG)
    sds = {k: {n: _r(v) for n, v in po.synthetic_state_dict(cfg, seed=s).items()} for k, s in
           (("student", 0), ("teacher", 1), ("ema", 2))}
    student = _model(cfg, sds["student"], torch.float32).train()
    student.y_embedder.uncond_prob = 0.0
    if checkpoint:
        from pixart_sigma_b200 import set_grad_checkpoint
        set_grad_checkpoint(student)
    teacher = _model(cfg, sds["teacher"]).eval()
    teacher.output_dtype = torch.float32
    ema = _model(cfg, sds["ema"], torch.float32).eval()
    ema.output_dtype = torch.float32
    red = GradBucketReducer(student)
    dist = LCMDistiller(student, red, teacher=teacher, ema=ema, loss_type=loss_type)
    latents, _, y, mask, _ = train_inputs(cfg, 2, (32, 32), [0, 0], [300, 41])
    g = torch.Generator().manual_seed(91)
    noise = torch.randn(latents.shape, generator=g)
    index = torch.tensor([0, 37])
    return cfg, sds, dist, red, (latents, y, mask, noise, index)


@pytest.mark.parametrize("loss_type", ["huber", "l2"])
def test_distillation_step_matches_oracle(loss_type):
    cfg, sds, dist, red, (latents, y, mask, noise, index) = _distill_setup(loss_type)
    red.zero_grad()
    loss = dist.step(latents.to(DEV), _r(y).to(DEV), mask.to(DEV), noise=noise.to(DEV), index=index.to(DEV))
    sdo = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sds["student"].items()}
    student = lambda x, t, yy, m: po.forward_grad(sdo, cfg, x, t.float(), yy, mask=m)
    inf = lambda sd: (lambda x, t, yy, m: po.forward(sd, cfg, _r(x), t.float(), yy, mask=m))
    uncond = _r(sds["student"]["y_embedder.y_embedding"]).repeat(2, 1, 1, 1)
    r = lo.distill_step(student, inf(sds["teacher"]), inf(sds["ema"]), latents, _r(y), mask, noise, index, uncond)
    want = r["loss_huber" if loss_type == "huber" else "loss_l2"]
    want.backward()
    e_loss = abs(float(loss) - float(want)) / abs(float(want))
    errs = {n: po.rel_err(p.grad.float().cpu(), sdo[n].grad) for n, p in dist.student.named_parameters()}
    worst = max(errs, key=errs.get)
    _log(f"lcm distillation step {loss_type} vs oracle: loss {float(loss):.6g} rel {e_loss:.2e}; grads max rel "
         f"{errs[worst]:.2e} ({worst})")
    # Huber with c = 1e-3 and |d| ~ 10 makes dl/dd = d / sqrt(d^2 + c^2) a sign per element: weight gradients are sums of
    # +-1-weighted terms that largely cancel, which magnifies the bf16 rounding of the forward by that cancellation; the
    # bound is then test_training_gpu.py's bound against the reference fixtures (3e-2).  L2 keeps the oracle bound 2e-2.
    assert e_loss < 2e-3 and errs[worst] < (3e-2 if loss_type == "huber" else 2e-2)


def test_batched_teacher_equals_two_forwards():
    cfg = po.OracleConfig(**CFG)
    m = _model(cfg, {k: _r(v) for k, v in po.synthetic_state_dict(cfg, seed=1).items()}).eval()
    m.output_dtype = torch.float32
    x, t, y, mask = po.synthetic_inputs(cfg, 2, (32, 32), lens=[300, 41])
    u = torch.randn_like(y)
    x, t, y, mask, u = x.to(DEV), t.to(DEV), y.to(DEV), mask.to(DEV), u.to(DEV)
    with torch.no_grad():
        both = m(torch.cat([x, x]), torch.cat([t, t]), torch.cat([y, u]), mask=torch.cat([mask, mask]))
        a, b = m(x, t, y, mask=mask), m(x, t, u, mask=mask)
    err = max(_rel(both[:2], a), _rel(both[2:], b))
    sd = {k: _r(v) for k, v in po.synthetic_state_dict(cfg, seed=1).items()}
    want = torch.cat([po.forward(sd, cfg, _r(x.cpu()), t.cpu(), _r(yy.cpu()), mask=mask.cpu()) for yy in (y, u)])
    e_or = max(_rel(both, want), _rel(torch.cat([a, b]), want))
    _log(f"batched teacher (2b) vs two batch-b forwards: rel {err:.2e}, bitwise {torch.equal(both, torch.cat([a, b]))}; "
         f"both vs oracle {e_or:.2e}")
    # the GEMMs pick their tiling / split-K by the row count, so bf16 activations can round differently at 2b and at b: the
    # two forms agree to bf16 level, and each is as close to the oracle as the smoke() bar requires
    assert err < 5e-3 and e_or < 1e-2


def test_ema_forward_sees_update_eager_and_graphed():
    cfg, sds, dist, red, (latents, y, mask, noise, index) = _distill_setup()
    x, t = latents.to(DEV), torch.tensor([5, 600], device=DEV)
    yy, mm = _r(y).to(DEV), mask.to(DEV)
    graphed = GraphedForward(dist.ema, method="forward")
    with torch.no_grad():
        before = graphed(x, t, yy, mm)
        for p in dist.student.parameters():                   # an optimizer step
            p.add_(0.05 * torch.randn_like(p))
        dist.update_ema()
        eager = dist.ema(x, t, yy, mask=mm)
        replay = graphed(x, t, yy, mm)
    fresh = _model(cfg, {k: v.to(torch.bfloat16) for k, v in dist.ema_state_dict().items()}).eval()
    fresh.output_dtype = torch.float32
    with torch.no_grad():
        want = fresh(x, t, yy, mask=mm)
    changed = _rel(before, want)
    _log(f"EMA forward after update_ema: changed by {changed:.2e}; eager equal {torch.equal(eager, want)}, "
         f"graphed equal {torch.equal(replay, want)}")
    assert changed > 1e-4 and torch.equal(eager, want) and torch.equal(replay, want)
    dist.ema.fuse_ln_modulate = True                          # derived weight copies keyed on _version: refused
    with pytest.raises(RuntimeError, match="fuse_ln_modulate"):
        dist.step(latents.to(DEV), yy, mm, noise=noise.to(DEV), index=index.to(DEV))


def test_eager_step_has_no_host_sync():
    _, _, dist, red, (latents, y, mask, noise, index) = _distill_setup()
    args = (latents.to(DEV), _r(y).to(DEV), mask.to(DEV))
    red.zero_grad()
    dist.step(*args)                                          # warm-up (workspaces, tables)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        red.zero_grad()
        loss = dist.step(*args)
        dist.update_ema()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    _log(f"eager distillation step without host sync: loss {float(loss):.4g}")
    assert torch.isfinite(loss)


@pytest.mark.parametrize("ckpt", [False, True])
def test_graphed_step_equals_eager(ckpt):
    runs = []
    for graphed in (False, True):
        _, _, dist, red, batch = _distill_setup(checkpoint=ckpt)
        batch = [v.to(DEV) for v in batch]
        batch[1] = _r(batch[1])
        opt = FlatCAME(red, lr=1e-5)
        update = lambda: (clip_grad_norm_(red, 0.01), opt.step())
        losses = []
        if graphed:
            step = GraphedLCMStep(dist, batch, optimizer_step=update)
            for _ in range(2):
                losses.append(step(*batch).clone())
        else:
            for _ in range(2):
                red.zero_grad()
                losses.append(dist.step(batch[0], batch[1], batch[2], noise=batch[3], index=batch[4]))
                update()
                dist.update_ema()
        torch.cuda.synchronize()
        runs.append((losses, [m.clone() for m in dist.master], [b["flat_param"].clone() for b in red.buckets]))
    (le, me, pe), (lg, mg, pg) = runs
    el = max(abs(float(a) - float(b)) / abs(float(a)) for a, b in zip(le, lg))
    em = max(_rel(b, a) for a, b in zip(me, mg))
    ep = max(_rel(b, a) for a, b in zip(pe, pg))
    _log(f"graphed LCM step vs eager (2 steps with clip + CAME + EMA): loss rel {el:.2e}, EMA master rel {em:.2e}, "
         f"student rel {ep:.2e}")
    assert el < 1e-4 and em < 1e-4 and ep < 1e-4
