"""LCM benchmark on PixArtMS-XL/2 (synthetic seeded weights): the 4-step LCM sampling loop at the c3 image shapes (4 images,
1024 px, batch 4, 300 caption tokens), eager and replayed from one CUDA graph; one consistency-distillation step at 1024 px
(student fp32 + gradient checkpointing, bf16 teacher and EMA) eager and graphed, with CUDA-event shares of its parts; and
`pxa_ema_flat` against the reference's `ema_update` loop (per-tensor mul_ / add_, then the bf16 cast the EMA forward needs)
on the XL/2 parameter set.  Prints one JSON line, with the card (name, power limit, max SM clock) read in the same run.

    python bench_lcm.py [--steps 3] [--warmup 1] [--distill-batch 2]
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

EMA_BYTES, EMA_REF_BYTES = 14, 34      # per parameter: fused pass; mul_ + scalar mul + add_ (28) and the bf16 cast (6)


def xl2(dtype, checkpoint=False):
    from pixart_sigma_b200 import build_model
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = build_model(dict(type="PixArtMS", depth=28, input_size=128, model_max_length=300), use_grad_checkpoint=checkpoint)
    return m.to(dtype)


def inputs(b, gen):
    x = torch.randn(b, 4, 128, 128, device="cuda", generator=gen)
    y = torch.randn(b, 1, 300, 4096, device="cuda", generator=gen).to(torch.bfloat16)
    mask = torch.ones(b, 300, dtype=torch.long, device="cuda")
    mask[1::2, 120:] = 0
    return x, y, mask


def bench_sampler(res, steps, warmup, gen):
    from pixart_sigma_b200 import lib
    from pixart_sigma_b200.lcm import LCMSampler
    m = xl2(torch.bfloat16).eval()
    m.output_dtype = torch.float32
    x, y, mask = inputs(4, gen)
    sampler = LCMSampler(m)
    kw = dict(y=y, mask=mask)
    for graph in (False, True):
        ms = timed(lambda: sampler.sample(x, steps=4, model_kwargs=kw, cuda_graph=graph), steps, warmup)
        n0 = lib.launch_count()
        sampler.sample(x, steps=4, model_kwargs=kw, cuda_graph=graph)
        torch.cuda.synchronize()
        res[f"sampler_4step_{'graphed' if graph else 'eager'}_ms"] = round(ms, 2)
        res[f"sampler_{'graphed' if graph else 'eager'}_lib_launches_per_step"] = (lib.launch_count() - n0) / 4
    del m, sampler
    torch.cuda.empty_cache()


def event_shares(student, red, dist, update, x, y, mask, b):
    """CUDA-event times of the parts of one instrumented eager step (the same calls as LCMDistiller._forward_loss).  A function
    of its own: the autograd graph of these steps must be gone before a step is captured, since the parameters' cached
    gradient accumulators keep the stream they were created on."""
    from pixart_sigma_b200 import autograd as ag
    from pixart_sigma_b200 import lcm, lib
    from pixart_sigma_b200.sampler import _step_input
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(8)]
    for _ in range(2):
        red.zero_grad()
        noise, index = dist.draw(x)
        start = dist.ddim_timesteps[index]
        t = (start - dist.topk).clamp_min(0)
        ev[0].record()
        x_t = dist.loss_fn.q_sample(x, start, noise).contiguous()
        ag.refresh_shadows(student)
        red.start()
        out_s = student(x_t, start, y, mask=mask)
        ev[1].record()
        with torch.no_grad():
            uncond = dist.uncond.to(dtype=y.dtype).expand(b, 1, *dist.uncond.shape)
            out_t = dist.teacher(torch.cat([x_t, x_t]), torch.cat([start, start]), torch.cat([y, uncond]), mask=torch.cat([mask, mask]))
            x_prev = torch.empty_like(x_t)
            lib.lcm_teacher_target(_step_input(out_t), x_t, index, dist.table, x_prev, w=dist.w)
            ev[2].record()
            out_e = dist.ema(x_prev, t, y, mask=mask)
        ev[3].record()
        loss = lcm._ConsistencyLoss.apply(out_s, _step_input(out_e), x_t, x_prev, index, dist.table, dist.partials,
                                          dist.loss_type, dist.huber_c)
        ev[4].record()
        loss.backward()
        red.finish()
        ev[5].record()
        update()
        ev[6].record()
        dist.update_ema()
        ev[7].record()
    torch.cuda.synchronize()
    span = lambda i, j: ev[i].elapsed_time(ev[j])
    parts = {"student_fwd_bwd": span(0, 1) + span(4, 5), "teacher_2b_fwd_and_target": span(1, 2), "ema_fwd": span(2, 3),
             "loss": span(3, 4), "clip_came": span(5, 6), "ema_update": span(6, 7)}
    total = sum(parts.values())
    return {k: round(v, 2) for k, v in parts.items()}, {k: round(v / total, 4) for k, v in parts.items()}


def bench_distill(res, steps, warmup, b, gen):
    from pixart_sigma_b200 import lcm
    from pixart_sigma_b200.optim import FlatCAME, clip_grad_norm_
    from pixart_sigma_b200.parallel import GradBucketReducer
    student = xl2(torch.float32, checkpoint=True).train()
    red = GradBucketReducer(student)
    dist = lcm.LCMDistiller(student, red)
    opt = FlatCAME(red, lr=1e-5)
    x, y, mask = inputs(b, gen)
    update = lambda: (clip_grad_norm_(red, 0.01), opt.step())

    def eager():
        red.zero_grad()
        dist.step(x, y, mask)
        update()
        dist.update_ema()
    res["distill_batch"] = b
    res["distill_eager_ms"] = round(timed(eager, steps, warmup), 1)
    res["distill_parts_ms"], res["distill_parts_share"] = event_shares(student, red, dist, update, x, y, mask, b)
    batch = (x, y, mask) + dist.draw(x)
    graphed = lcm.GraphedLCMStep(dist, batch, optimizer_step=update)
    res["distill_graphed_ms"] = round(timed(lambda: graphed(*batch), steps, warmup), 1)
    del graphed
    return student, red, dist


def bench_ema(res, steps, warmup, student, red, dist):
    n = sum(sum(p.numel() for p in bk["params"]) for bk in red.buckets)
    ms = timed(dist.update_ema, max(steps, 10), warmup)
    ema_params = dict(dist.ema.named_parameters())
    pairs = [(m[o:o + int(torch.Size(s).numel())].view(s), p) for m, lay, bk in zip(dist.master, dist.layout, red.buckets)
             for (name, o, s), p in zip(lay, bk["params"])]
    shadows = [ema_params[name] for lay in dist.layout for name, _, _ in lay]

    def reference():                                       # train_pixart_lcm.py:48-53, then the EMA model's bf16 copy
        with torch.no_grad():
            for d, s in pairs:
                d.mul_(0.95).add_((1 - 0.95) * s.data)
            for (d, _), h in zip(pairs, shadows):
                h.copy_(d)
    ms_ref = timed(reference, max(steps, 10), warmup)
    res["ema_params"] = n
    res["ema_flat_ms"], res["ema_flat_gbps"] = round(ms, 3), round(n * EMA_BYTES / ms / 1e6, 1)
    res["ema_reference_loop_ms"], res["ema_reference_loop_gbps"] = round(ms_ref, 3), round(n * EMA_REF_BYTES / ms_ref / 1e6, 1)
    res["ema_bytes_per_param"] = {"ema_flat": EMA_BYTES, "reference_loop": EMA_REF_BYTES}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--distill-batch", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lcm.py measures on a GPU"
    res = {"bench": "lcm", "card": card()}
    gen = torch.Generator(device="cuda").manual_seed(0)
    bench_sampler(res, args.steps, args.warmup, gen)
    student, red, dist = bench_distill(res, args.steps, args.warmup, args.distill_batch, gen)
    bench_ema(res, args.steps, args.warmup, student, red, dist)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
