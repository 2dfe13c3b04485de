#!/usr/bin/env python
"""bench_dora.py -- DoRA fine-tuning against LoRA on the native training path (one JSON line).

    python bench_dora.py [--steps K] [--warmup W] [--rank R]

Step = bench_lora.py's step (`training.train_step` with `DDPMEpsLoss`, activation checkpointing on every block,
`clip_grad_norm_(reducer, 1.0)`, `FlatAdamW.step()`), eager, CUDA-event timed, at bench_lora.py's two shapes (PixArt XL/2
512px batch 16 with 120 caption tokens; Sigma XL/2 1024px batch 2 with 300 tokens), with a rank-R adapter on every target of
the reference script: LoRA (`inject_lora`) and DoRA (`inject_dora`), with the peak allocated memory of each.

DoRA kernel times, from one extra instrumented step whose `pxa_dora_norm` and `pxa_dora_bwd` calls are bracketed by CUDA
events: `norm_ms` = every pxa_dora_norm launch of the step (the per-step c = m / ||W + s B A||), `bwd_ms` = every pxa_dora_bwd
call (dz = c g and the magnitude gradient), with the bytes each moves and the rate that gives.  `merge_ms`: `merge_lora` of
the DoRA adapter on the XL/2 parameter set (host clock around a device synchronise; it includes the copy of the replaced
weights to the host).  Card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench_lora as bl  # noqa: E402  (shapes, batch, step and timer of the LoRA benchmark)


def _model(shape, rank, dora):
    from pixart_sigma_b200 import build_model, lora
    kw = dict(type="PixArtMS", depth=28, input_size=shape["latent"], pe_interpolation=shape["pe"],
              model_max_length=shape["tokens"], class_dropout_prob=0.0)
    with torch.device("cuda"):
        m = build_model(kw, use_grad_checkpoint=True)
    m = m.float().train()
    with torch.no_grad():                         # the initialisation zeroes some projections: zero-norm rows for DoRA
        for p in m.parameters():
            if p.dim() >= 2 and not bool(p.any()):
                p.normal_(0, 0.02)
    (lora.inject_dora if dora else lora.inject_lora)(m, rank, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():                         # a trained-looking adapter (fresh B is zero, fresh c is one)
        for _, mod in lora._adapted(m):
            mod.lora_B.normal_(0, 0.01)
            if dora:
                mod.lora_magnitude.mul_(1.01)
    return m


def _dora_kernels(step, batch):
    """ms and bytes of every pxa_dora_norm / pxa_dora_bwd call of one instrumented step."""
    from pixart_sigma_b200 import lib
    acc = {"norm": [], "bwd": []}
    nbytes = {"norm": 0, "bwd": 0}
    norm, bwd = lib.dora_norm, lib.dora_bwd

    def timed(kind, fn, *a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(*a, **kw)
        e1.record()
        acc[kind].append((e0, e1))

    def n(items, *, N, K, T):
        nbytes["norm"] += len(items) * (N * K * 2 + (N + K) * T * 2 + N * 8)
        timed("norm", norm, items, N=N, K=K, T=T)

    def b(g, y, bias, c, m, dz, dm):
        nbytes["bwd"] += 3 * g.numel() * 2 + 2 * ((g.shape[0] + lib.DORA_BWD_ROWS - 1) // lib.DORA_BWD_ROWS) * g.shape[1] * 4
        timed("bwd", bwd, g, y, bias, c, m, dz, dm)
        return dz

    lib.dora_norm, lib.dora_bwd = n, b
    try:
        step(batch)
        torch.cuda.synchronize()
    finally:
        lib.dora_norm, lib.dora_bwd = norm, bwd
    out = {}
    for k, v in acc.items():
        ms = sum(a.elapsed_time(z) for a, z in v)
        out[k] = {"ms": round(ms, 3), "calls": len(v), "gbytes": round(nbytes[k] / 1e9, 3),
                  "tb_per_s": round(nbytes[k] / (ms * 1e-3) / 1e12, 3) if ms > 0 else None}
    return out


def _merge_ms(m):
    from pixart_sigma_b200 import lora
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    lora.merge_lora(m)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    lora.unmerge_lora(m)
    return round(ms, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rank", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dora.py needs a CUDA device")
    torch.cuda.set_device(0)
    name, power = bl._card()
    line = {"metric": "dora_step_ms", "gpu": name, "power_limit_w": power, "rank": args.rank, "steps": args.steps}
    for tag, shape in bl.SHAPES.items():
        batch = bl._batch(shape)
        for mode in ("lora", "dora"):
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            m = _model(shape, args.rank, mode == "dora")
            step = bl._stepper(m)
            ms = bl._time(lambda: step(batch), args.steps, args.warmup)
            entry = {"step_ms": round(ms, 2), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                     "trained_params": sum(p.numel() for p in m.parameters() if p.requires_grad)}
            if mode == "dora":
                entry["kernels"] = _dora_kernels(step, batch)
                if tag == "alpha512":
                    entry["merge_ms"] = _merge_ms(m)
            line[f"{tag}_{mode}"] = entry
            del m, step
        line[f"{tag}_dora_over_lora"] = round(line[f"{tag}_dora"]["step_ms"] / line[f"{tag}_lora"]["step_ms"] - 1, 4)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
