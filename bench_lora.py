#!/usr/bin/env python
"""bench_lora.py -- LoRA fine-tuning against full fine-tuning on the native training path (one JSON line).

    python bench_lora.py [--steps K] [--warmup W] [--rank R] [--skip-full]

Step = `training.train_step` with `DDPMEpsLoss` (forward + backward, activation checkpointing on every block) +
`clip_grad_norm_(reducer, 1.0)` + `FlatAdamW(lr=1e-5, weight_decay=1e-2, eps=1e-8).step()`, eager, CUDA-event timed, at the
shapes of the reference's LoRA launch script and of Sigma's 1024px config:
  alpha512   PixArt XL/2 512px (64 x 64 latents, 1024 tokens), batch 16, 120 caption tokens
  sigma1024  PixArt-Sigma XL/2 1024px (128 x 128 latents, 4096 tokens), batch 2, 300 caption tokens
each with a rank-R adapter on every target of the script (`lora.TARGET_MODULES`) and as a full fine-tuning step (every
parameter trained), with the peak allocated memory of each.

Shares of a LoRA step, from one extra instrumented step whose GEMM calls are bracketed by CUDA events (so the shares are of
that step's summed kernel time, not of the uninstrumented step): `tail` = the extra time of every K-tail GEMM over the same
call without its tail (the call is repeated into a scratch output), `skinny` = the down-projections u = x A^T, v = s dY B and
the adapter weight gradients dA, dB, `prep` = `lora.prepare_operands`.

`gemm_c3`: the six GEMMs of a c3 block (8 x 4096 rows; qkv, attn proj, cross q, cross proj, fc1 with the GELU-aux epilogue,
fc2; the projections' gated fp32 residual epilogues) with a rank-16 tail against `pxa_gemm_bf16`, alternated call by call in
one process, median of the per-round times.  Card name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SHAPES = {"alpha512": dict(latent=64, batch=16, tokens=120, pe=1.0), "sigma1024": dict(latent=128, batch=2, tokens=300, pe=2.0)}


def _card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                      text=True).strip().split(",")
        return out[0].strip(), float(out[1])
    except (OSError, subprocess.CalledProcessError, ValueError, IndexError):
        return torch.cuda.get_device_name(0), None


def _model(shape, rank):
    from pixart_sigma_b200 import build_model, lora
    kw = dict(type="PixArtMS", depth=28, input_size=shape["latent"], pe_interpolation=shape["pe"],
              model_max_length=shape["tokens"], class_dropout_prob=0.0)
    with torch.device("cuda"):
        m = build_model(kw, use_grad_checkpoint=True)
    m = m.float().train()
    if rank:
        lora.inject_lora(m, rank, generator=torch.Generator().manual_seed(0))
        with torch.no_grad():                     # a trained-looking adapter (fresh B is zero)
            for _, mod in lora._adapted(m):
                mod.lora_B.normal_(0, 0.01)
    return m


def _batch(shape):
    g = torch.Generator(device="cuda").manual_seed(1)
    B, h, L = shape["batch"], shape["latent"], shape["tokens"]
    x0 = torch.randn(B, 4, h, h, device="cuda", generator=g)
    y = torch.randn(B, 1, L, 4096, device="cuda", generator=g).to(torch.bfloat16).float()
    mask = torch.ones(B, L, dtype=torch.long, device="cuda")
    t = torch.randint(0, 1000, (B,), device="cuda", generator=g)
    return x0, t, y, mask, torch.randn(x0.shape, device="cuda", generator=g)


def _stepper(m):
    from pixart_sigma_b200.optim import FlatAdamW, clip_grad_norm_
    from pixart_sigma_b200.parallel import GradBucketReducer
    from pixart_sigma_b200.training import DDPMEpsLoss, train_step
    red = GradBucketReducer(m)
    opt = FlatAdamW(red, lr=1e-5, weight_decay=1e-2, eps=1e-8)
    loss = DDPMEpsLoss()

    def step(batch):
        x0, t, y, mask, noise = batch
        red.zero_grad()
        train_step(m, loss, x0, t, y, mask, noise=noise, reducer=red)
        clip_grad_norm_(red, 1.0)
        opt.step()
    return step


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in ev)


def _shares(m, step, batch):
    """One instrumented LoRA step: ms of the tail overhead, the skinny adapter GEMMs and the operand preparation."""
    from pixart_sigma_b200 import lib, lora
    acc = {"tail": [], "skinny": [], "prep": [], "all": []}
    gemm, wgrad, prep = lib.gemm, lib.gemm_wgrad, lora.prepare_operands

    def timed(kind, fn, *a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn(*a, **kw)
        e1.record()
        acc[kind].append((e0, e1))
        return r

    adapter_ops = set()

    def g(a, w, bias, out, **kw):
        if w.data_ptr() in adapter_ops:
            return timed("skinny", gemm, a, w, bias, out, **kw)
        if kw.get("tail_a") is not None:
            r = timed("all", gemm, a, w, bias, out, **kw)
            plain = {k: v for k, v in kw.items() if k not in ("tail_a", "tail_w")}
            if plain.get("out_aux") is not None:
                plain["out_aux"] = torch.empty_like(plain["out_aux"])
            timed("tail", gemm, a, w, bias, torch.empty_like(out), **plain)     # subtracted below
            return r
        return gemm(a, w, bias, out, **kw)

    def wg(a_t, w_t, out, **kw):                  # adapter weight gradients: M = T rows
        return timed("skinny", wgrad, a_t, w_t, out, **kw) if out.shape[0] < 128 else wgrad(a_t, w_t, out, **kw)

    def p(model):
        timed("prep", prep, model)
        adapter_ops.clear()
        for mod in model.modules():
            op = mod.__dict__.get("_pxa_lora")
            if op is not None:
                adapter_ops.update((op.a.data_ptr(), op.bt.data_ptr()))

    lib.gemm, lib.gemm_wgrad, lora.prepare_operands = g, wg, p
    try:
        step(batch)
        torch.cuda.synchronize()
    finally:
        lib.gemm, lib.gemm_wgrad, lora.prepare_operands = gemm, wgrad, prep
    ms = {k: sum(a.elapsed_time(b) for a, b in v) for k, v in acc.items()}
    return {"tail": ms["all"] - ms["tail"], "skinny": ms["skinny"], "prep": ms["prep"]}


def _gemm_c3(rank, rounds):
    """The six c3 block GEMMs with a rank-`rank` tail against pxa_gemm_bf16, alternated per round."""
    from pixart_sigma_b200 import lib
    M, C, B = 8 * 4096, 1152, 8
    bf = dict(dtype=torch.bfloat16, device="cuda")
    r = lambda *s: torch.randn(*s, **bf) * 0.05
    x32 = torch.randn(M, C, device="cuda")
    gate = torch.randn(B, 6, C, device="cuda")
    gk = dict(gate=gate[:, 2], gate_batch_stride=gate.stride(0), rows_per_batch=4096)
    aux = torch.empty(M, C, **bf)
    calls = {   # name: (a, w, out, T, kwargs)
        "qkv": (r(M, C), r(3 * C, C), torch.empty(M, 3 * C, **bf), 3 * rank, {}),
        "proj": (r(M, C), r(C, C), torch.empty(M, C, device="cuda"), rank,
                 dict(epilogue=lib.EPI_BIAS_RESIDUAL, residual=x32, out_aux=aux, aux_is_branch=True, **gk)),
        "q": (r(M, C), r(C, C), torch.empty(M, C, **bf), rank, {}),
        "cproj": (r(M, C), r(C, C), torch.empty(M, C, device="cuda"), rank,
                  dict(epilogue=lib.EPI_BIAS_RESIDUAL, residual=x32, rows_per_batch=4096)),
        "fc1": (r(M, C), r(4 * C, C), torch.empty(M, 4 * C, **bf), rank,
                dict(epilogue=lib.EPI_BIAS_GELU_AUX, out_aux=torch.empty(M, 4 * C, **bf))),
        "fc2": (r(M, 4 * C), r(C, 4 * C), torch.empty(M, C, device="cuda"), rank,
                dict(epilogue=lib.EPI_BIAS_RESIDUAL, residual=x32, out_aux=aux, aux_is_branch=True, **gk)),
    }
    res = {}
    for name, (a, w, out, T, kw) in calls.items():
        bias = r(w.shape[0])
        ta, tw = r(M, T), r(w.shape[0], T)
        fns = {"plain": lambda: lib.gemm(a, w, bias, out, **kw), "tail": lambda: lib.gemm(a, w, bias, out, tail_a=ta, tail_w=tw, **kw)}
        for f in fns.values():
            for _ in range(3):
                f()
        t = {k: [] for k in fns}
        for _ in range(rounds):
            for k, f in fns.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(5):
                    f()
                e1.record()
                t[k].append((e0, e1))
        torch.cuda.synchronize()
        res[name] = {k: round(statistics.median(a.elapsed_time(b) / 5 for a, b in v), 4) for k, v in t.items()}
    tot = {k: round(sum(v[k] for v in res.values()), 4) for k in ("plain", "tail")}
    return {"per_gemm_ms": res, "total_ms": tot, "tail_overhead": round(tot["tail"] / tot["plain"] - 1, 4), "T_base": rank}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rank", type=int, default=16)
    ap.add_argument("--skip-full", action="store_true", help="only the LoRA steps (no full fine-tuning comparison)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lora.py needs a CUDA device")
    torch.cuda.set_device(0)
    name, power = _card()
    line = {"metric": "lora_step_ms", "gpu": name, "power_limit_w": power, "rank": args.rank, "steps": args.steps}
    for tag, shape in SHAPES.items():
        batch = _batch(shape)
        for mode in ("lora",) + (() if args.skip_full else ("full",)):
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            m = _model(shape, args.rank if mode == "lora" else 0)
            step = _stepper(m)
            ms = _time(lambda: step(batch), args.steps, args.warmup)
            entry = {"step_ms": round(ms, 2), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                     "trained_params": sum(p.numel() for p in m.parameters() if p.requires_grad)}
            if mode == "lora":
                sh = _shares(m, step, batch)
                total = sum(sh.values())
                entry["instrumented_ms"] = {k: round(v, 2) for k, v in sh.items()}
                entry["share_of_step"] = {k: round(v / ms, 4) for k, v in sh.items()}
                entry["share_total"] = round(total / ms, 4)
            line[f"{tag}_{mode}"] = entry
            del m, step
    line["gemm_c3"] = _gemm_c3(args.rank, rounds=10)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
