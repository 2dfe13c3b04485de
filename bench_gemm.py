"""GEMM benchmark at the six calls of one PixArt-Sigma-XL/2 block of the c3 workload (1024px, batch 8: M = 32768 tokens,
rows_per_batch 4096, hidden 1152), with the epilogues, gates, aux outputs and tile order model.py gives them.

For each call it times, alternating in one process on one card:
  bn0        `pxa_gemm_bf16` with block_n 0 (the library's automatic schedule choice)
  bn192      the same call with block_n 192 (the cooperative 128 x 192 schedule)
  bn0_bias   / bn192_bias: the same product with the cheapest epilogue (EPI_BIAS, bf16 out); for the fp32 residual calls the
             difference to the real call is what the epilogue costs
  cublas     torch.matmul of the same bf16 operands: cuBLAS on the same card as the attainable plain-GEMM rate (a measurement
             only; nothing in the library uses it)
and reports ms, TFLOP/s, the minimum HBM bytes of the call with the resulting GB/s, and which floor (989 TFLOP/s dense BF16 or
3.35 TB/s HBM3, data-sheet H100 SXM figures) bounds the call together with the call's share of it.  Prints a table on stderr and
one JSON line on stdout, with the card (name, power limit, max SM clock) read in the same run.

    python bench_gemm.py [--seconds 0.5] [--rounds 3]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_optim import card  # noqa: E402

PEAK_TFLOPS, PEAK_GBS = 989.0, 3350.0
B, T, C, MLP = 8, 4096, 1152, 4608
M = B * T


def make_calls(lib):
    """name -> (N, K, call(block_n, cheap)); the residual calls write x32 in place like model.py does."""
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, device="cuda", generator=g) * scale)
    x32 = rnd(M, C)
    xb = torch.empty(M, C, dtype=torch.bfloat16, device="cuda")
    mod = rnd(B, 6, C, scale=0.1)                              # gate rows of the adaLN-single modulation, per sample
    ms = mod.stride(0)
    a_c = rnd(M, C).to(torch.bfloat16)                         # inputs of the K = 1152 calls
    a_h = rnd(M, MLP).to(torch.bfloat16)                       # hidden activations (fc2 input)
    w = {(n, k): (rnd(n, k, scale=k ** -0.5).to(torch.bfloat16), rnd(n, scale=0.1).to(torch.bfloat16))
         for n, k in ((3 * C, C), (C, C), (MLP, C), (C, MLP))}
    outs = {n: torch.empty(M, n, dtype=torch.bfloat16, device="cuda") for n in (C, 3 * C, MLP)}

    def call(a, n, k, **kw):
        wt, bias = w[(n, k)]

        def run(block_n, cheap):
            if cheap:
                lib.gemm(a, wt, bias, outs[n], epilogue=lib.EPI_BIAS, block_n=block_n)
            elif kw.get("epilogue") == lib.EPI_BIAS_RESIDUAL:
                lib.gemm(a, wt, bias, x32, residual=x32, block_n=block_n, **kw)
            else:
                lib.gemm(a, wt, bias, outs[n], block_n=block_n, **kw)
        return (a, wt), run

    res = dict(epilogue=lib.EPI_BIAS_RESIDUAL)
    return {
        "attn.qkv": (3 * C, C, "bias, bf16", *call(a_c, 3 * C, C)),
        "attn.proj": (C, C, "fp32 residual + gate + bf16 aux",
                      *call(a_c, C, C, gate=mod[:, 2], gate_batch_stride=ms, rows_per_batch=T, out_aux=xb, **res)),
        "cross.q_linear": (C, C, "bias, bf16", *call(a_c, C, C)),
        "cross.proj": (C, C, "fp32 residual", *call(a_c, C, C, **res)),
        "mlp.fc1": (MLP, C, "bias + GELU, bf16", *call(a_c, MLP, C, epilogue=lib.EPI_BIAS_GELU)),
        "mlp.fc2": (C, MLP, "fp32 residual + gate",
                    *call(a_h, C, MLP, gate=mod[:, 5], gate_batch_stride=ms, rows_per_batch=T, reverse_tiles=True, **res)),
    }


def min_bytes(n, k, epi):
    """A and W read once, outputs written once, the fp32 residual read once."""
    b = M * k * 2 + n * k * 2
    if epi.startswith("fp32 residual"):
        b += M * n * 4 * 2 + (M * n * 2 if "aux" in epi else 0)
    else:
        b += M * n * 2
    return b


def time_window(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5, help="timed launches per variant and shape, in seconds (over all rounds)")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds over the variants; the median round is reported")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gemm.py measures on a GPU"
    from pixart_sigma_b200 import lib

    calls = make_calls(lib)
    rows = []
    for name, (n, k, epi, (a, wt), run) in calls.items():
        variants = {
            "bn0": lambda: run(0, False),
            "bn192": lambda: run(192, False),
            "bn0_bias": lambda: run(0, True),
            "bn192_bias": lambda: run(192, True),
            "cublas": lambda: torch.matmul(a, wt.t()),
        }
        iters = {}
        for v, fn in variants.items():                         # warm-up, then size each window from a short timing
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            iters[v] = max(5, int(args.seconds / args.rounds / (time_window(fn, 5) * 1e-3)))
        times = {v: [] for v in variants}
        for _ in range(args.rounds):
            for v, fn in variants.items():
                times[v].append(time_window(fn, iters[v]))
        flop = 2.0 * M * n * k
        nbytes = min_bytes(n, k, epi)
        mma_ms, hbm_ms = flop / (PEAK_TFLOPS * 1e12) * 1e3, nbytes / (PEAK_GBS * 1e9) * 1e3
        row = {"call": name, "M": M, "N": n, "K": k, "epilogue": epi, "min_bytes": nbytes,
               "bound": "MMA" if mma_ms >= hbm_ms else "HBM", "floor_ms": round(max(mma_ms, hbm_ms), 4)}
        for v in variants:
            ms = sorted(times[v])[len(times[v]) // 2]
            vb = min_bytes(n, k, "bias, bf16") if v.endswith("_bias") or v == "cublas" else nbytes
            row[v] = {"ms": round(ms, 4), "tflops": round(flop / (ms * 1e-3) / 1e12, 1), "gbs": round(vb / (ms * 1e-3) / 1e9, 1),
                      "share_of_floor": round(max(mma_ms, hbm_ms) / ms, 3), "spread_ms": round(max(times[v]) - min(times[v]), 4)}
        rows.append(row)
        print(f"{name:15s} N {n:5d} K {k:5d} {row['bound']} floor {row['floor_ms']:.3f} ms | " +
              " | ".join(f"{v} {row[v]['ms']:.3f} ms {row[v]['tflops']:.0f} TF/s" for v in variants), file=sys.stderr)
    tot = {v: round(sum(r[v]["ms"] for r in rows), 4) for v in ("bn0", "bn192", "cublas")}
    print(json.dumps({"workload": "c3 block GEMMs (M 32768, rows_per_batch 4096)", "calls": rows, "block_total_ms": tot,
                      "gpu": card()}))


if __name__ == "__main__":
    main()
