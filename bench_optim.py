"""Optimizer-step benchmark on the PixArtMS-XL/2 parameter set (610.9 M fp32 parameters in 29 reducer buckets, seeded random
gradients): gradient clipping + `FlatCAME.step` (eager and replayed from one CUDA graph), `FlatAdamW.step`, and the plain-torch
clip + CAME loop of oracle/came_oracle.py, which stands in for the came_pytorch path a reference user runs.  Prints one JSON
line: CUDA-event times per step, library launches per step, optimizer state bytes, achieved GB/s from the bytes each pass
structure moves, and the card (name, power limit, max SM clock) read in the same run.

    python bench_optim.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CLIP_BYTES, CAME_BYTES, ADAMW_BYTES = 12, 32, 28          # HBM bytes per parameter of each pass structure


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(out[0]), float(out[1])
    except Exception as exc:                                   # noqa: BLE001 -- report, do not fail the measurement
        info["nvidia_smi"] = f"unavailable: {exc}"
    return info


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_optim.py measures on a GPU"
    from oracle import came_oracle as co
    from pixart_sigma_b200 import PixArtMS_XL_2, lib
    from pixart_sigma_b200.optim import FlatAdamW, FlatCAME, clip_grad_norm_
    from pixart_sigma_b200.parallel import GradBucketReducer

    torch.manual_seed(0)
    with torch.device("cuda"):
        model = PixArtMS_XL_2(input_size=128)
    red = GradBucketReducer(model)
    n = sum(p.numel() for p in model.parameters())
    for p in model.parameters():
        p.grad.normal_().mul_(1e-3)
    came = FlatCAME(red)                                   # Sigma config: lr 2e-5, betas (0.9, 0.999, 0.9999), eps (1e-30, 1e-16)
    adamw = FlatAdamW(red)

    def clip_came():
        clip_grad_norm_(red, 0.01)
        came.step()

    n0 = lib.launch_count()
    clip_came()
    torch.cuda.synchronize()
    launches = lib.launch_count() - n0
    res = {"model": "PixArtMS_XL_2 (input_size=128)", "params": n, "buckets": len(red.buckets), "steps": args.steps,
           "came_launches_per_step": launches}
    res["clip_ms"] = timed(lambda: clip_grad_norm_(red, 0.01), args.steps, args.warmup)
    res["came_step_ms"] = timed(came.step, args.steps, args.warmup)
    res["clip_came_eager_ms"] = timed(clip_came, args.steps, args.warmup)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph):
            clip_came()
    torch.cuda.current_stream().wait_stream(side)
    res["clip_came_graph_ms"] = timed(graph.replay, args.steps, args.warmup)
    res["adamw_step_ms"] = timed(adamw.step, args.steps, args.warmup)

    params = list(model.parameters())
    states = [{} for _ in params]
    grads = [p.grad for p in params]

    def oracle():
        co.clip_grad_norm(grads, 0.01)
        co.came_step([p.data for p in params], grads, states, lr=2e-5)

    res["oracle_clip_came_ms"] = timed(oracle, max(args.steps // 4, 2), 1)
    res["came_state_bytes"] = came.state_bytes()
    res["adamw_state_bytes"] = sum(t.numel() * 4 for st in adamw.state for t in st.values())
    gbs = lambda nbytes, ms: round(nbytes * n / (ms * 1e-3) / 1e9, 1)
    res["clip_gb_s"] = gbs(CLIP_BYTES, res["clip_ms"])
    res["came_step_gb_s"] = gbs(CAME_BYTES, res["came_step_ms"])
    res["adamw_step_gb_s"] = gbs(ADAMW_BYTES, res["adamw_step_ms"])
    res["speedup_vs_oracle_graph"] = round(res["oracle_clip_came_ms"] / res["clip_came_graph_ms"], 1)
    for k in list(res):
        if k.endswith("_ms"):
            res[k] = round(res[k], 3)
    res["gpu"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
