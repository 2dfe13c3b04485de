"""Sampling-loop benchmark: the S = 25 SA-Solver loop (scripts/inference.py:119-133's call) next to the 20-step DPM-Solver++
loop (:102-118), eager and as one CUDA graph, around the full PixArt-Sigma-XL/2 denoiser at the c3 shapes of bench.py
(1024px, 4 images, forward batch 8 = CFG pairs, 300 caption tokens, synthetic bf16 weights built as bench.py builds them).
The IDDPM loop (:89-101: `IDDPM("100").p_sample_loop(model.forward_with_cfg, ..., clip_denoised=False)`, cfg 4.5) is timed
three ways on the same model: the torch loop (`p_sample_loop_progressive` driven to the end), and the native loop eager and
as one CUDA graph (with the capture time); `iddpm_native_vs_glue_rel_err` compares the native and the torch loop's samples
drawn from the same seed.

For each loop: wall time of one whole sampling run (CUDA events around work that ends in a synchronise, after a warm-up run
that also captures the graph), denoise-steps/s (images x evaluations / s), library kernel launches per evaluation (eager), and
the sampler overhead = loop time - evaluations x the time of one eager forward (10 back to back) measured in the same process;
within run-to-run noise that difference can come out slightly negative.  The card name,
power limit and max SM clock are read (read-only) in the same run.  Prints one JSON line.

    python bench_sampling.py [--reps 3] [--images 4] [--side 128] [--iddpm-steps 100]
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

L = 300


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                   # noqa: BLE001 -- reported, not fatal
        return {"name": torch.cuda.get_device_name(), "power_limit": None, "max_sm_clock": None, "error": repr(e)}


def timed_ms(fn, reps: int) -> float:
    """Median over `reps` runs of CUDA-event time around fn(), each ending in a synchronise."""
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--side", type=int, default=128, help="latent side (128 = 1024px)")
    ap.add_argument("--depth", type=int, default=28)
    ap.add_argument("--iddpm-steps", type=int, default=100, help="IDDPM respacing (scripts/inference.py's default: 100)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampling.py measures on the GPU; no CUDA device found")
    from pixart_sigma_b200 import PixArtMS, SASolverSampler, lib
    from pixart_sigma_b200.iddpm import IDDPM
    from pixart_sigma_b200.sampler import DPMS

    dev = torch.device("cuda")
    imgs, side = args.images, args.side
    torch.manual_seed(1234)
    with torch.device(dev):
        model = PixArtMS(depth=args.depth, hidden_size=1152, patch_size=2, num_heads=16, input_size=side,
                         pe_interpolation=side / 64, model_max_length=L)
        for blk in model.blocks:                            # un-zero the zero-initialised layers, as bench.py does
            torch.nn.init.normal_(blk.cross_attn.proj.weight, std=0.02)
        torch.nn.init.normal_(model.final_layer.linear.weight, std=0.02)
    model = model.to(torch.bfloat16).eval()

    g = torch.Generator().manual_seed(99)
    z = torch.randn(imgs, 4, side, side, generator=g).to(dev)
    y = torch.randn(2 * imgs, 1, L, 4096, generator=g).to(torch.bfloat16).to(dev)
    lens = torch.randint(8, L + 1, (imgs,), generator=g)
    mask = (torch.arange(L)[None] < lens[:, None]).long().to(dev)
    null, cond = y[:imgs], y[imgs:]
    kw = dict(data_info=None, mask=mask)
    t = torch.full((2 * imgs,), 999.0, device=dev)
    x2 = torch.cat([z, z])

    res = {"gpu": gpu_info(), "images": imgs, "latent": [side, side], "forward_batch": 2 * imgs, "depth": args.depth}
    with torch.no_grad():
        model.forward_with_dpmsolver(x2, t, y, **kw)                         # warm-up
        n0 = lib.launch_count()
        model.forward_with_dpmsolver(x2, t, y, **kw)
        launches_fwd = lib.launch_count() - n0
        # back to back, as inside a sampling loop (a single forward between synchronises also times the launch ramp)
        fwd_ms = timed_ms(lambda: [model.forward_with_dpmsolver(x2, t, y, **kw) for _ in range(10)], args.reps) / 10
        res["forward"] = {"ms": fwd_ms, "launches": launches_fwd}

        sa = SASolverSampler(model.forward_with_dpmsolver, device="cuda")
        dpm = DPMS(model.forward_with_dpmsolver, condition=cond, uncondition=null, cfg_scale=4.5, model_kwargs=kw)
        loops = {
            "sa_solver_s25": (25, lambda graph: sa.sample(S=25, batch_size=imgs, shape=(4, side, side), eta=1, conditioning=cond,
                                                          unconditional_conditioning=null, unconditional_guidance_scale=4.5,
                                                          model_kwargs=kw, x_T=z, cuda_graph=graph)[0]),
            "dpm_solver_s20": (20, lambda graph: dpm.sample(z, steps=20, order=2, skip_type="time_uniform", method="multistep",
                                                            cuda_graph=graph)),
        }
        for name, (evals, run) in loops.items():
            for graph in (False, True):
                run(graph)                                                   # warm-up (and capture)
                n0 = lib.launch_count()
                if not graph:
                    run(False)
                    torch.cuda.synchronize()
                launches = (lib.launch_count() - n0) / evals if not graph else None
                ms = timed_ms(lambda: run(graph), args.reps)
                res[f"{name}_{'graph' if graph else 'eager'}"] = {
                    "evaluations": evals, "ms": round(ms, 2), "denoise_steps_per_s": round(imgs * evals / (ms / 1000.0), 3),
                    "launches_per_step": launches, "overhead_ms": round(ms - evals * fwd_ms, 2),
                    "overhead_ms_per_step": round((ms - evals * fwd_ms) / evals, 3)}

        # IDDPM as scripts/inference.py:89-101 runs it: the n latents repeated to the 2n CFG batch, y = [caption ; null]
        steps = args.iddpm_steps
        iddpm = IDDPM(str(steps))
        z2 = z.repeat(2, 1, 1, 1)
        ikw = dict(y=torch.cat([cond, null]), cfg_scale=4.5, data_info=None, mask=mask)
        icall = dict(clip_denoised=False, model_kwargs=ikw, device=dev)

        def glue():
            for out in iddpm.p_sample_loop_progressive(model.forward_with_cfg, z2.shape, z2, **icall):
                pass
            return out["sample"]
        iloops = {"glue": glue,
                  "eager": lambda: iddpm.p_sample_loop(model.forward_with_cfg, z2.shape, z2, **icall),
                  "graph": lambda: iddpm.p_sample_loop(model.forward_with_cfg, z2.shape, z2, cuda_graph=True, **icall)}
        samples = {}
        for form, run in iloops.items():
            torch.cuda.manual_seed(5)
            samples[form] = run()                                             # warm-up (and capture), seeded
            n0 = lib.launch_count()
            if form != "graph":
                run()
                torch.cuda.synchronize()
            launches = (lib.launch_count() - n0) / steps if form != "graph" else None
            ms = timed_ms(run, args.reps)
            entry = {"evaluations": steps, "ms": round(ms, 2), "denoise_steps_per_s": round(imgs * steps / (ms / 1000.0), 3),
                     "launches_per_step": launches, "overhead_ms": round(ms - steps * fwd_ms, 2),
                     "overhead_ms_per_step": round((ms - steps * fwd_ms) / steps, 3)}
            if form == "graph":
                entry["capture_s"] = round(iddpm.last_capture_s, 2)
            res[f"iddpm_s{steps}_{form}"] = entry
        ref = samples["glue"].double()
        res["iddpm_native_vs_glue_rel_err"] = {
            form: float((samples[form].double() - ref).norm() / ref.norm()) for form in ("eager", "graph")}
    res["forward"]["ms"] = round(fwd_ms, 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
