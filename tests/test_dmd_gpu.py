"""GPU tests (-m gpu) of the DMD kernel and drivers (pixart_sigma_b200/dmd.py) against fp64 formulas, the oracle
(oracle/dmd_oracle.py) and the reference fixtures (tests/golden/dmd_*.pt).  Each test prints its measured error (shown with
`pytest -rP` or `-s`).

Tolerances:
  * pxa_dmd_loss vs fp64: loss 1e-6 relative, gradient 1e-5, weight 1e-6 (fp32 operations rounded as the reference's);
  * the fake model's denoising loss (`_eps_mse`) vs fp64 F.mse_loss: loss 1e-6, gradient 1e-6;
  * sampler with the toy denoiser vs the reference fixtures: 1e-5; around a depth-2 PixArtMS vs the oracle on the same
    bf16-rounded weights: 2e-2 (bf16 GEMM operands);
  * full step vs the oracle (same bf16-rounded weights): loss 2e-3, gradients 2e-2, the bounds of test_training_gpu.py,
    scaled for the real == fake == generator case by the cancellation in score_fake - score_real (see the test);
  * EMA vs diffusers' update: 1e-6 relative (the two forms differ only in rounding).
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dmd_oracle as dmo            # noqa: E402
from oracle import dpm_oracle as do             # noqa: E402
from oracle import pixart_oracle as po          # noqa: E402
from oracle.gen_golden_dmd import CFG, SAMPLE_CASES, STEP_CASES, step_inputs  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"

if torch.cuda.is_available():
    from pixart_sigma_b200 import build_model, lib
    from pixart_sigma_b200.dmd import DMDDistiller, DMDSampler, ddpm_alphas_cumprod, dmd_draws, ema_decay
    from pixart_sigma_b200.optim import FlatAdamW, clip_grad_norm_
    from pixart_sigma_b200.parallel import GradBucketReducer


def _log(line):
    print(line)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _gold(name):
    return torch.load(os.path.join(GOLD, name + ".pt"))


def _r(v):
    return v.to(torch.bfloat16).float()


# ------------------------------------------------------------------------------------------------- kernel
def _f64_dm(latents, noisy, t, ac, real_out, fake_out, cfg, sa_g, sb_g):
    """The reference's arithmetic (train_pixart_dmd.py:538-561) in fp64 on the same fp32 inputs."""
    b = latents.shape[0]
    a = ac.double()[t].view(-1, 1, 1, 1)
    sa, sb = a.sqrt(), (1 - a).sqrt()
    su, sc = (-real_out[:, :4].double()).chunk(2)
    sr = su + cfg * (sc - su)
    coeff = (-fake_out[:, :4].double() - sr) * sb / sa
    pred = (noisy.double() + sb * sr) / sa
    lat = latents.double()
    weight = 1.0 / ((lat - pred).abs().mean([1, 2, 3], keepdim=True) + 1e-5)
    d = lat - (lat - weight * coeff)
    n = d.numel()
    grad = torch.zeros(b, 8, *latents.shape[2:], dtype=torch.float64, device=latents.device)
    grad[:, :4] = (2 * d / n) / sa_g * (-sb_g)
    return (d ** 2).mean(), grad, weight.reshape(b)


def _kernel_inputs(dtype, t):
    g = torch.Generator().manual_seed(4)
    b, h, w = len(t), 16, 20
    ac = ddpm_alphas_cumprod().to(DEV)
    t = torch.tensor(t, dtype=torch.long, device=DEV)
    latents = torch.randn(b, 4, h, w, generator=g).to(DEV)
    noise = torch.randn(b, 4, h, w, generator=g).to(DEV)
    tc = t.clamp(0, 999)
    noisy = (ac[tc].sqrt().view(-1, 1, 1, 1) * latents + (1 - ac[tc]).sqrt().view(-1, 1, 1, 1) * noise).contiguous()
    real = torch.randn(2 * b, 8, h, w, generator=g).to(dtype).to(DEV)
    fake = torch.randn(b, 8, h, w, generator=g).to(dtype).to(DEV)
    return latents, noisy, t, ac, real, fake


def _launch(latents, noisy, t, ac, real, fake, out_channels=8):
    b = latents.shape[0]
    d = torch.full((b, out_channels) + tuple(latents.shape[2:]), 7.0, device=DEV)
    loss, weight = torch.empty((), device=DEV), torch.empty(b, device=DEV)
    partials = torch.empty(2 * b * lib.DMD_PARTS, dtype=torch.float64, device=DEV)
    lib.dmd_loss(latents, noisy, t, ac, real[:, :4], fake[:, :4], d, loss, weight, partials, cfg=3.0,
                 gen_sqrt_alpha=0.0063527, gen_sqrt_beta=0.99998)
    return loss, d, weight


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_dmd_loss_kernel_matches_fp64(dtype):
    inp = _kernel_inputs(dtype, [2, 500, 995])
    runs = [_launch(*inp) for _ in range(2)]
    same = all(torch.equal(a, b) for a, b in zip(runs[0], runs[1]))                         # bitwise reproducible
    loss, d, weight = runs[0]
    ref_loss, ref_grad, ref_w = _f64_dm(*inp, 3.0, 0.0063527, 0.99998)
    e_loss = abs(float(loss) - float(ref_loss)) / float(ref_loss)
    e_grad, e_w = _rel(d, ref_grad), _rel(weight, ref_w)
    sigma_zero = bool((d[:, 4:] == 0).all())
    _log(f"pxa_dmd_loss {dtype}: loss rel {e_loss:.2e}, grad rel {e_grad:.2e}, weight rel {e_w:.2e}, sigma channels zero "
         f"{sigma_zero}, two launches bitwise equal {same}")
    assert e_loss < 1e-6 and e_grad < 1e-5 and e_w < 1e-6 and sigma_zero and same
    d4 = _launch(*inp, out_channels=4)[1]                                                    # a 4-channel generator output
    assert torch.equal(d4, d[:, :4])


def test_dmd_loss_out_of_range_timestep_stays_in_its_sample():
    inp = _kernel_inputs(torch.float32, [2, 1000, 995])
    loss, d, weight = _launch(*inp)
    ok_loss, ok_d, ok_w = _launch(*_kernel_inputs(torch.float32, [2, 500, 995]))
    keep = [0, 2]
    contained = (bool(torch.isnan(weight[1])) and bool(torch.isnan(d[1, :4]).all()) and bool((d[1, 4:] == 0).all())
                 and torch.equal(weight[keep], ok_w[keep]) and torch.equal(d[keep], ok_d[keep]))
    _log(f"pxa_dmd_loss with t = 1000 in sample 1: weight {weight.tolist()}, loss {float(loss)}, other samples unchanged "
         f"{contained}")
    assert contained and torch.isnan(loss)


# ------------------------------------------------------------------------------------------------- sampler
def _model(cfg, sd, dtype=torch.bfloat16):
    kw = dict(type="PixArtMS", depth=cfg.depth, hidden_size=cfg.hidden_size, num_heads=cfg.num_heads, input_size=cfg.input_size,
              pe_interpolation=cfg.pe_interpolation, model_max_length=cfg.model_max_length, class_dropout_prob=0.0)
    with torch.device(DEV):
        m = build_model(kw)
    m.load_state_dict(sd, strict=False)
    return m.to(dtype)


@pytest.mark.parametrize("name", sorted(n for n, c in SAMPLE_CASES.items() if c["model"] == "toy"))
def test_sampler_with_toy_denoiser_matches_reference_fixture(name):
    gd = _gold(name)
    sampler = DMDSampler(do.toy_model, timestep=gd["case"]["t"])
    kw = dict(cond=gd["cond"].to(DEV))
    eager = sampler.sample(gd["x_T"].to(DEV), model_kwargs=kw)
    graphed = [sampler.sample(gd["x_T"].to(DEV), model_kwargs=kw, cuda_graph=True) for _ in range(2)]
    err = _rel(eager, gd["out"])
    same = all(torch.equal(g, eager) for g in graphed)
    _log(f"dmd sampler {name}: rel err vs reference {err:.2e}, graph replays equal eager {same}")
    assert err < 1e-5 and same


@pytest.mark.parametrize("t", [400, 999])
def test_sampler_around_pixartms_matches_oracle(t):
    gd = _gold(f"dmd_sample_d2_t{t}")
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    sd = {k: _r(v) for k, v in po.synthetic_state_dict(cfg, seed=0).items()}
    m = _model(cfg, sd).eval()
    m.output_dtype = torch.float32
    _, _, y, mask = po.synthetic_inputs(cfg, 2, (32, 32), lens=[300, 77])
    x = gd["x_T"]
    sampler = DMDSampler(m, timestep=t)
    kw = dict(y=_r(y).to(DEV), mask=mask.to(DEV))
    got = sampler.sample(x.to(DEV), model_kwargs=kw)
    graphed = sampler.sample(x.to(DEV), model_kwargs=kw, cuda_graph=True)
    want = dmo.sample(lambda xx, tt: po.forward(sd, cfg, _r(xx), tt.float(), _r(y), mask=mask), x, t)
    err, e_gold = _rel(got, want), _rel(got, gd["out"])
    _log(f"dmd sampler around PixArtMS depth 2, t={t}: rel err vs oracle {err:.2e} (vs the fp32 reference fixture "
         f"{e_gold:.2e}), graph replay equal eager {torch.equal(graphed, got)}")
    assert err < 2e-2 and torch.equal(graphed, got)


# ------------------------------------------------------------------------------------------------- distiller
def _setup(name="dmd_step_d2"):
    gd = _gold(name)
    cfg = po.OracleConfig(**CFG)
    sds = {k: {n: _r(v) for n, v in po.synthetic_state_dict(cfg, seed=s).items()} for k, s in gd["seeds"].items()}
    gen = _model(cfg, sds["generator"], torch.float32).train()
    fake = _model(cfg, sds["fake"], torch.float32).train()
    real = _model(cfg, sds["real"]).eval()
    real.output_dtype = torch.float32
    ema = _model(cfg, sds["ema"], torch.float32).eval()
    ema.output_dtype = torch.float32
    gred, fred = GradBucketReducer(gen), GradBucketReducer(fake)
    y, mask, uy, um = step_inputs(cfg, 2, gd["lens"])
    dist = DMDDistiller(gen, gred, fake, fred, _r(uy).to(DEV), um.to(DEV), real=real, ema=ema)
    torch.manual_seed(gd["rng"])                             # the reference's draws, regenerated on the CPU generator
    draws = tuple(v.to(DEV) for v in dmd_draws(2, (cfg.input_size,) * 2, "cpu"))
    return gd, cfg, sds, dist, (_r(y)[:, None].to(DEV), mask.to(DEV)), draws, (uy, um)


def test_eps_mse_matches_fp64():
    _, _, _, dist, _, _, _ = _setup()
    g = torch.Generator().manual_seed(6)
    out = torch.randn(3, 8, 16, 20, generator=g).to(DEV).requires_grad_(True)
    target = torch.randn(3, 4, 16, 20, generator=g).to(DEV)
    loss = dist._eps_mse(out, target)
    loss.backward()
    o64 = out.detach().double().requires_grad_(True)
    ref = F.mse_loss(o64[:, :4], target.double())
    ref.backward()
    e_loss, e_grad = abs(float(loss.detach()) - float(ref)) / float(ref), _rel(out.grad, o64.grad)
    _log(f"_eps_mse vs fp64 F.mse_loss: loss rel {e_loss:.2e}, grad rel {e_grad:.2e}, sigma grads zero "
         f"{bool((out.grad[:, 4:] == 0).all())}")
    assert e_loss < 1e-6 and e_grad < 1e-6 and bool((out.grad[:, 4:] == 0).all())


@pytest.mark.parametrize("name", sorted(STEP_CASES))
def test_step_matches_oracle(name):
    gd, cfg, sds, dist, (y, mask), draws, (uy, um) = _setup(name)
    dist.gen_reducer.zero_grad()
    dist.fake_reducer.zero_grad()
    dm, sg = dist.step(y, mask, draws=draws)
    step_fake = {n: p.grad.clone() for n, p in dist.fake.named_parameters()}
    sdo = {k: {n: v.clone().requires_grad_(k in ("generator", "fake")) for n, v in sd.items()} for k, sd in sds.items()}
    train = lambda sd: (lambda x, t, yy, m: po.forward_grad(sd, cfg, x, t.float(), yy, mask=m))
    inf = lambda sd: (lambda x, t, yy, m: po.forward(sd, cfg, _r(x), t.float(), yy, mask=m))   # bf16 x: the kernels' input
    r = dmo.step(train(sdo["generator"]), inf(sdo["real"]), train(sdo["fake"]), y.cpu(), mask.cpu(), _r(uy)[:, None], um,
                 tuple(v.cpu() for v in draws))
    r["dm_loss"].backward()
    # The fake model's step is checked on latents at the scale of VAE latents (unit rms), with the same draws.  The step's
    # own latents are the x0 of an untrained synthetic generator at t = 999, where sqrt(1 - a) / sqrt(a) ~ 157 makes them
    # ~170 in magnitude.  PixArt's cross-attention reads the un-normalised residual stream, so its logits grow with the input
    # and the bf16 q operand's rounding grows with them: the cross-attention q_linear gradient of ANY training step on such
    # inputs leaves the range test_training_gpu.py's 2e-2 bound covers (printed below as "fake grads on the step's latents").
    # The fake reducer holding exactly this loss's gradient is test_fake_reducer_holds_only_the_denoising_gradient.
    _, _, _, noise_f, t_f = draws
    lat1 = (dist.latents / dist.latents.pow(2).mean().sqrt()).contiguous()
    dist.fake_reducer.zero_grad()
    dist.fake_reducer.start()
    dist._eps_mse(dist.fake(dist.add_noise(lat1, noise_f, t_f), t_f, y, mask=mask), noise_f.contiguous()).backward()
    out_f = train(sdo["fake"])(dmo.add_noise(dmo.alphas_cumprod(), lat1.cpu(), noise_f.cpu(), t_f.cpu()), t_f.cpu(), y.cpu(),
                               mask.cpu())
    F.mse_loss(out_f[:, :4].float(), noise_f.cpu()).backward()
    sdo_step = {n: v.clone().requires_grad_(True) for n, v in sds["fake"].items()}
    out_s = train(sdo_step)(dmo.add_noise(dmo.alphas_cumprod(), dist.latents.cpu(), noise_f.cpu(), t_f.cpu()), t_f.cpu(),
                            y.cpu(), mask.cpu())
    F.mse_loss(out_s[:, :4].float(), noise_f.cpu()).backward()
    e_dm = abs(float(dm) - float(r["dm_loss"].detach())) / float(r["dm_loss"].detach())
    e_sg = abs(float(sg) - float(r["sg_loss"].detach())) / float(r["sg_loss"].detach())
    e_lat, e_w = _rel(dist.latents, r["latents"].detach()), _rel(dist.weight, r["weight"])
    errs = {}
    for which, model in (("generator", dist.generator), ("fake", dist.fake)):
        for n, p in model.named_parameters():
            errs[f"{which}.{n}"] = po.rel_err(p.grad.float().cpu(), sdo[which][n].grad)
    wg = max((k for k in errs if k.startswith("generator.")), key=errs.get)
    wf = max((k for k in errs if k.startswith("fake.")), key=errs.get)
    e_step = max(po.rel_err(g.float().cpu(), sdo_step[n].grad) for n, g in step_fake.items())
    # coeff = (score_fake - score_real) sb / sa is a difference: an error of relative size e in the model outputs becomes
    # e * kappa in coeff (and in the gradient it scales), kappa = (|score_fake| + |score_real|) / |score_fake - score_real|.
    # With distinct models kappa is O(1); with real == fake == generator (the recipe's start) score_fake cancels the
    # conditional part of score_real and only the guidance term (cfg - 1)(eps_c - eps_u) is left, so the oracle bounds of
    # test_training_gpu.py (2e-3 loss, 2e-2 gradients) apply to the un-cancelled terms and are scaled by kappa.
    su, sc = (-r["real_out"][:, :4]).chunk(2)
    s_real, s_fake = su + 3.0 * (sc - su), -r["fake_out"][:, :4]
    kappa = float((s_fake.norm() + s_real.norm()) / (s_fake - s_real).norm())
    scale = kappa if name.endswith("_same") else 1.0
    _log(f"dmd step {name} vs oracle: dm_loss {float(dm):.6g} rel {e_dm:.2e}, sg_loss {float(sg):.6g} rel {e_sg:.2e}, "
         f"latents rel {e_lat:.2e}, weight rel {e_w:.2e}, generator grads max rel {errs[wg]:.2e} ({wg}), fake grads max rel "
         f"{errs[wf]:.2e} ({wf}) (on the step's latents {e_step:.2e}); kappa {kappa:.2f}, bound scale {scale:.2f}")
    assert e_dm < 2e-3 * scale and e_sg < 2e-3 and errs[wg] < 2e-2 * scale and errs[wf] < 2e-2


def test_fake_reducer_holds_only_the_denoising_gradient():
    gd, cfg, sds, dist, (y, mask), draws, _ = _setup()
    for red in (dist.gen_reducer, dist.fake_reducer):
        red.zero_grad()
    dist.step(y, mask, draws=draws)
    after_step = [b["flat"].clone() for b in dist.fake_reducer.buckets]
    dist.fake_reducer.zero_grad()
    _, _, _, noise_f, t_f = draws
    out_f = dist.fake(dist.add_noise(dist.latents, noise_f, t_f), t_f, y, mask=mask)
    dist._eps_mse(out_f, noise_f.contiguous()).backward()
    alone = [b["flat"] for b in dist.fake_reducer.buckets]
    err = max(_rel(a, b) for a, b in zip(after_step, alone))
    _log(f"fake reducer after a step vs the denoising loss alone: rel {err:.2e}")
    assert err < 1e-4                       # the reorder tolerance of test_training_gpu.py (atomics in the backward)


def test_step_has_no_host_sync():
    _, _, _, dist, (y, mask), _, _ = _setup()
    for red in (dist.gen_reducer, dist.fake_reducer):
        red.zero_grad()
    dist.step(y, mask)                                       # warm-up (workspaces)
    gopt, fopt = FlatAdamW(dist.gen_reducer, lr=1e-5, eps=1e-6), FlatAdamW(dist.fake_reducer, lr=1e-5, eps=1e-6)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for red in (dist.gen_reducer, dist.fake_reducer):
            red.zero_grad()
        dm, sg = dist.step(y, mask)
        clip_grad_norm_(dist.gen_reducer, 1.0)
        gopt.step()
        clip_grad_norm_(dist.fake_reducer, 1.0)
        fopt.step()
        dist.update_ema()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    _log(f"DMD step without host sync: dm_loss {float(dm):.4g}, sg_loss {float(sg):.4g}")
    assert torch.isfinite(dm) and torch.isfinite(sg)


def test_training_iteration_with_adamw_clip_and_ema():
    _, _, _, dist, (y, mask), draws, _ = _setup()
    gopt, fopt = FlatAdamW(dist.gen_reducer, lr=1e-4, eps=1e-6), FlatAdamW(dist.fake_reducer, lr=1e-4, eps=1e-6)
    gen0 = [b["flat_param"].clone() for b in dist.gen_reducer.buckets]
    fake0 = [b["flat_param"].clone() for b in dist.fake_reducer.buckets]
    losses, e_ema = [], []
    for it in range(2):
        for red in (dist.gen_reducer, dist.fake_reducer):
            red.zero_grad()
        losses += list(dist.step(y, mask, draws=draws if it == 0 else None))
        clip_grad_norm_(dist.gen_reducer, 1.0)
        gopt.step()
        clip_grad_norm_(dist.fake_reducer, 1.0)
        fopt.step()
        before = [m.clone() for m in dist._flat_ema.master]
        dist.update_ema()
        decay = ema_decay(it + 1)
        for m, m0, b in zip(dist._flat_ema.master, before, dist.gen_reducer.buckets):
            n = sum(p.numel() for p in b["params"])
            want = m0[:n].double().clone()
            want -= (1 - decay) * (want - b["flat_param"][:n].double())          # diffusers' form, fp64
            e_ema.append(_rel(m[:n], want))
    moved = min(_rel(b["flat_param"], p0) for b, p0 in zip(dist.gen_reducer.buckets, gen0))
    moved_f = min(_rel(b["flat_param"], p0) for b, p0 in zip(dist.fake_reducer.buckets, fake0))
    first_equal = dist.ema_updates == 2
    _log(f"DMD iteration x2 (clip + AdamW for both models, EMA): losses {[round(float(v), 5) for v in losses]}, generator "
         f"moved {moved:.2e}, fake moved {moved_f:.2e}, EMA vs diffusers' update max rel {max(e_ema):.2e}")
    assert all(torch.isfinite(v) for v in losses) and moved > 0 and moved_f > 0 and first_equal and max(e_ema) < 1e-6
    sd = dist.ema_state_dict()
    assert all(v.dtype == torch.float32 for k, v in sd.items() if k in dict(dist.generator.named_parameters()))
