"""DMD benchmark on PixArtMS-XL/2 (synthetic seeded weights): one distribution-matching distillation step, eager, with
CUDA-event shares of its parts and the peak memory, at the recipe's shape (PixArt-alpha XL/2 at 512 px: 64 x 64 latents, 120
caption tokens, batch 4) and at Sigma 1024 px (128 x 128 latents, 300 tokens, batch 2); one-step sampling at the c3 shapes
(4 images, 1024 px, batch 4, 300 tokens) eager and replayed from a CUDA graph; and `pxa_dmd_loss` against a plain-torch
restatement of train_pixart_dmd.py:519-561.  Prints one JSON line, with the card (name, power limit, max SM clock) read in
the same run.

    python bench_dmd.py [--steps 3] [--warmup 1]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from bench_optim import card, timed  # noqa: E402

SHAPES = {"alpha_512_b4": dict(input_size=64, tokens=120, pe_interpolation=1.0, batch=4),
          "sigma_1024_b2": dict(input_size=128, tokens=300, pe_interpolation=2.0, batch=2)}


def xl2(shape, dtype, checkpoint=False):
    from pixart_sigma_b200 import build_model
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = build_model(dict(type="PixArtMS", depth=28, input_size=shape["input_size"], model_max_length=shape["tokens"],
                             pe_interpolation=shape["pe_interpolation"], class_dropout_prob=0.0),
                        use_grad_checkpoint=checkpoint)
    return m.to(dtype)


def captions(b, tokens, gen):
    y = torch.randn(b, 1, tokens, 4096, device="cuda", generator=gen).to(torch.bfloat16)
    mask = torch.ones(b, tokens, dtype=torch.long, device="cuda")
    mask[1::2, tokens // 3:] = 0
    return y, mask


def event_shares(dist, b, y, mask, update_gen, update_fake):
    """CUDA-event times of the parts of one instrumented eager step: the calls of DMDDistiller.step, split at the events."""
    from pixart_sigma_b200 import autograd as ag
    from pixart_sigma_b200 import lib
    from pixart_sigma_b200.dmd import _DmdLoss
    from pixart_sigma_b200.capture import step_input
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(11)]
    for _ in range(2):
        for red in (dist.gen_reducer, dist.fake_reducer):
            red.zero_grad()
        init_noise, noise, t, noise_f, t_f = dist.draw(b)
        partials, weight, _ = dist._workspace(b)
        dist.gen_reducer.start()
        dist.fake_reducer.start()
        ev[0].record()
        ag.refresh_shadows(dist.generator)
        out_g = dist.generator(init_noise, torch.full((b,), dist.one_step_t, device="cuda"), y, mask=mask)
        ev[1].record()
        with torch.no_grad():
            latents, scratch = torch.empty_like(init_noise), torch.empty_like(init_noise)
            lib.lcm_step(step_input(out_g[:, :4]), init_noise, None, latents, scratch, **dist.gen_scalars)
            noisy = dist.add_noise(latents, noise, t).contiguous()
            uy = dist.uncond_y.to(dtype=y.dtype).expand(b, *dist.uncond_y.shape[1:])
            m2 = torch.cat([dist.uncond_mask.to(mask.dtype).expand(b, -1), mask])
            real_out = dist.real(torch.cat([noisy, noisy]), torch.cat([t, t]), torch.cat([uy, y]), mask=m2)
        ev[2].record()
        ag.refresh_shadows(dist.fake)
        fake_out = dist.fake(noisy, t, y, mask=mask).detach()
        ev[3].record()
        dm = _DmdLoss.apply(out_g, latents, noisy, t, dist.ac, step_input(real_out), step_input(fake_out), partials, weight,
                            dist.cfg, dist.gen_scalars["sqrt_alpha"], dist.gen_scalars["sqrt_beta"])
        ev[4].record()
        dm.backward()
        ev[5].record()
        del fake_out, real_out
        out_f = dist.fake(dist.add_noise(latents, noise_f, t_f), t_f, y, mask=mask)
        dist._eps_mse(out_f, noise_f).backward()
        ev[6].record()
        update_gen()
        ev[7].record()
        update_fake()
        ev[8].record()
        dist.update_ema()
        ev[9].record()
    torch.cuda.synchronize()
    span = lambda i, j: ev[i].elapsed_time(ev[j])
    parts = {"generator_fwd_bwd": span(0, 1) + span(4, 5), "real_2b_fwd": span(1, 2), "fake_dm_fwd": span(2, 3),
             "dmd_loss_kernels": span(3, 4), "fake_fwd_bwd": span(5, 6), "gen_clip_adamw": span(6, 7),
             "fake_clip_adamw": span(7, 8), "ema_update": span(8, 9)}
    total = sum(parts.values())
    return {k: round(v, 2) for k, v in parts.items()}, {k: round(v / total, 4) for k, v in parts.items()}


def bench_step(res, name, shape, steps, warmup, gen):
    from pixart_sigma_b200.dmd import DMDDistiller
    from pixart_sigma_b200.optim import FlatAdamW, clip_grad_norm_
    from pixart_sigma_b200.parallel import GradBucketReducer
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    b, L = shape["batch"], shape["tokens"]
    generator = xl2(shape, torch.float32, checkpoint=True).train()
    fake = xl2(shape, torch.float32, checkpoint=True).train()
    gred, fred = GradBucketReducer(generator), GradBucketReducer(fake)
    uy = torch.randn(1, 1, L, 4096, device="cuda", generator=gen).to(torch.bfloat16)
    um = torch.zeros(1, L, dtype=torch.long, device="cuda")
    um[0, 0] = 1
    dist = DMDDistiller(generator, gred, fake, fred, uy, um)
    gopt, fopt = FlatAdamW(gred, lr=1e-5, eps=1e-6), FlatAdamW(fred, lr=1e-5, eps=1e-6)
    y, mask = captions(b, L, gen)
    update_gen = lambda: (clip_grad_norm_(gred, 1.0), gopt.step())
    update_fake = lambda: (clip_grad_norm_(fred, 1.0), fopt.step())

    def eager():
        gred.zero_grad()
        fred.zero_grad()
        dist.step(y, mask)
        update_gen()
        update_fake()
        dist.update_ema()
    r = {"batch": b, "latent": shape["input_size"], "tokens": L, "eager_ms": round(timed(eager, steps, warmup), 1)}
    r["parts_ms"], r["parts_share"] = event_shares(dist, b, y, mask, update_gen, update_fake)
    r["peak_mem_gb"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    res[f"step_{name}"] = r
    del dist, generator, fake, gred, fred, gopt, fopt
    torch.cuda.empty_cache()


def bench_sampler(res, steps, warmup, gen):
    from pixart_sigma_b200 import lib
    from pixart_sigma_b200.dmd import DMDSampler
    m = xl2(SHAPES["sigma_1024_b2"], torch.bfloat16).eval()
    m.output_dtype = torch.float32
    x = torch.randn(4, 4, 128, 128, device="cuda", generator=gen)
    y, mask = captions(4, 300, gen)
    sampler = DMDSampler(m, timestep=400)
    kw = dict(y=y, mask=mask)
    for graph in (False, True):
        tag = "graphed" if graph else "eager"
        res[f"sampler_1step_{tag}_ms"] = round(timed(lambda: sampler.sample(x, model_kwargs=kw, cuda_graph=graph), max(steps, 5),
                                                     warmup), 2)
        n0 = lib.launch_count()
        sampler.sample(x, model_kwargs=kw, cuda_graph=graph)
        torch.cuda.synchronize()
        res[f"sampler_{tag}_lib_launches"] = lib.launch_count() - n0
    del m, sampler
    torch.cuda.empty_cache()


def bench_loss(res, steps, warmup, gen):
    """pxa_dmd_loss vs the reference's torch glue (train_pixart_dmd.py:538-561 plus the eps_to_mu backward) at the Sigma
    1024 px step shape, fp32 model outputs."""
    from pixart_sigma_b200 import lib
    from pixart_sigma_b200.dmd import ddpm_alphas_cumprod
    b, h = 2, 128
    ac = ddpm_alphas_cumprod().cuda()
    t = torch.randint(1, 999, (b,), device="cuda", generator=gen)
    lat, noisy = (torch.randn(b, 4, h, h, device="cuda", generator=gen) for _ in range(2))
    real, fake = torch.randn(2 * b, 8, h, h, device="cuda", generator=gen), torch.randn(b, 8, h, h, device="cuda", generator=gen)
    d, loss, weight = torch.empty(b, 8, h, h, device="cuda"), torch.empty((), device="cuda"), torch.empty(b, device="cuda")
    partials = torch.empty(2 * b * lib.DMD_PARTS, dtype=torch.float64, device="cuda")
    kernel = lambda: lib.dmd_loss(lat, noisy, t, ac, real[:, :4], fake[:, :4], d, loss, weight, partials, cfg=3.0,
                                  gen_sqrt_alpha=0.0063527, gen_sqrt_beta=0.99998)
    lat_g = lat.clone().requires_grad_(True)

    def reference():
        su, sc = (-real[:, :4]).chunk(2)
        sr = su + 3.0 * (sc - su)
        a = ac[t]
        beta = 1.0 - a
        coeff = (-fake[:, :4] - sr) * beta.view(-1, 1, 1, 1) ** 0.5 / a.view(-1, 1, 1, 1) ** 0.5
        pred = (noisy + beta.view(-1, 1, 1, 1) ** 0.5 * sr) / a.view(-1, 1, 1, 1) ** 0.5
        w = 1. / ((lat_g - pred).abs().mean([1, 2, 3], keepdim=True) + 1e-5).detach()
        lv = torch.nn.functional.mse_loss(lat_g, (lat_g - w * coeff).detach())
        (g,) = torch.autograd.grad(lv, lat_g)
        torch.cat([g / 0.0063527 * -0.99998, torch.zeros_like(g)], dim=1)
    res["dmd_loss_shape"] = [b, 4, h, h]
    res["dmd_loss_kernel_ms"] = round(timed(kernel, max(steps, 20), warmup), 4)
    res["dmd_loss_torch_ms"] = round(timed(reference, max(steps, 20), warmup), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dmd.py measures on a GPU"
    res = {"bench": "dmd", "card": card()}
    gen = torch.Generator(device="cuda").manual_seed(0)
    bench_loss(res, args.steps, args.warmup, gen)
    bench_sampler(res, args.steps, args.warmup, gen)
    for name, shape in SHAPES.items():
        bench_step(res, name, shape, args.steps, args.warmup, gen)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
