"""Attention-forward benchmark at the head_dim-72 calls of the flagship workloads, with the layouts model.py / autograd.py give them:

  c3.self    batch 8 (4 images, CFG pairs), 16 heads, 4096 x 4096, q / k / v strided views of the interleaved qkv GEMM output,
             samples taken last to first (reverse_batch, as model.py chains them through L2)
  c3.cross   the same queries against the packed caption keys: batch 8, at most 300 keys per sample, with the ragged caption
             lengths bench.py draws for c3 (seed 99), repeated over the CFG pairs
  c4.full    batch 2, 16384 x 16384 from the interleaved qkv buffer (the 2K layers without KV compression)
  c4.kvc     batch 2, 16384 queries against 4096 compressed keys from separate K / V buffers (the KV-compressed layers)
  c5.self    the training forward: batch 4, 4096 x 4096, P as bf16 hi + lo terms (fp32_attention) and the lse output

For each call it times, alternating in one process on one card, `pxa_flash_attn_d72_bf16` and, as a yardstick, torch's
scaled_dot_product_attention on the same tensors with each backend that accepts them (nothing in the library uses it).  It
reports ms, the algorithmic rate (4 Nq Nk 72 FLOP per head and sample; the cross call counts the valid keys only), and the share
of the 989 TFLOP/s dense BF16 floor (H100 SXM data sheet).  Prints a table on stderr and one JSON line on stdout, with the card
(name, power limit, max SM clock) read in the same run.

    python bench_attn.py [--seconds 1.0] [--rounds 3] [--no-sdpa]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_optim import card  # noqa: E402

PEAK_TFLOPS = 989.0
H, D, C, L = 16, 72, 1152, 300


def c3_caption_lengths():
    """The caption lengths of bench.py's c3 run: its generator draws the latents and the captions first."""
    g = torch.Generator().manual_seed(99)
    torch.randn(8, 4, 128, 128, generator=g)
    torch.randn(8, 1, L, 4096, generator=g)
    lens = torch.randint(8, L + 1, (4,), generator=g)
    return torch.cat([lens, lens]).tolist()


def make_calls(lib):
    """name -> (description, FLOP, ours(), {backend: (q, k, v, mask)} for sdpa)."""
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g).to(torch.bfloat16)
    calls = {}

    def self_call(name, B, N, fp32_p=False, reverse=False):
        qkv = rnd(B * N, 3, H, D)
        out = torch.empty(B * N, H * D, dtype=torch.bfloat16, device="cuda")
        lse = torch.empty(B, H, N, dtype=torch.float32, device="cuda") if fp32_p else None
        st = (3 * H * D, D)

        def ours():
            lib.flash_attn(qkv[:, 0], qkv[:, 1], qkv[:, 2], out, B=B, H=H, Nq=N, Nk=N, kv_rows=B * N, q_strides=st, k_strides=st,
                           v_strides=st, lse=lse, reverse_batch=reverse, fp32_p=fp32_p)
        r = qkv.view(B, N, 3, H, D)
        sd = tuple(r[:, :, i].transpose(1, 2) for i in range(3)) + (None,)
        form = "bf16 hi + lo P, lse" if fp32_p else "bf16 P"
        calls[name] = (f"B {B}, {N} x {N}, interleaved qkv, {form}", 4.0 * B * H * N * N * D, ours, sd)

    def cross_call(lens):
        B, N = len(lens), 4096
        q = rnd(B * N, C)
        kv = rnd(sum(lens), 2 * C)
        out = torch.empty(B * N, C, dtype=torch.bfloat16, device="cuda")
        kv_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
        offs = [sum(lens[:i]) for i in range(B)]
        kv_off = torch.tensor(offs, dtype=torch.int32, device="cuda")
        kv4 = kv.view(-1, 2, H, D)

        def ours():
            lib.flash_attn(q, kv4[:, 0], kv4[:, 1], out, B=B, H=H, Nq=N, Nk=L, kv_rows=kv.shape[0], kv_len=kv_len, kv_off=kv_off,
                           q_strides=(C, D), k_strides=(2 * C, D), v_strides=(2 * C, D))
        kp = torch.zeros(B, L, 2, H, D, dtype=torch.bfloat16, device="cuda")  # padded copy with a key mask for sdpa
        for b, n in enumerate(lens):
            kp[b, :n] = kv4[offs[b]:offs[b] + n]
        mask = (torch.arange(L, device="cuda")[None] < kv_len[:, None]).view(B, 1, 1, L)
        calls["c3.cross"] = (f"B {B}, {N} x <= {L} packed keys, lengths {lens}", 4.0 * H * N * sum(lens) * D, ours,
                             (q.view(B, N, H, D).transpose(1, 2), kp[:, :, 0].transpose(1, 2), kp[:, :, 1].transpose(1, 2), mask))

    def kvc_call(B, N, Nk):
        qkv = rnd(B * N, 3 * C)
        kc, vc = rnd(B * Nk, C), rnd(B * Nk, C)
        out = torch.empty(B * N, C, dtype=torch.bfloat16, device="cuda")

        def ours():
            lib.flash_attn(qkv[:, :C], kc, vc, out, B=B, H=H, Nq=N, Nk=Nk, kv_rows=B * Nk, q_strides=(3 * C, D), k_strides=(C, D),
                           v_strides=(C, D), reverse_batch=True)
        calls["c4.kvc"] = (f"B {B}, {N} x {Nk}, compressed K / V buffers", 4.0 * B * H * N * Nk * D, ours,
                           (qkv.view(B, N, 3, H, D)[:, :, 0].transpose(1, 2), kc.view(B, Nk, H, D).transpose(1, 2),
                            vc.view(B, Nk, H, D).transpose(1, 2), None))

    self_call("c3.self", 8, 4096, reverse=True)
    cross_call(c3_caption_lengths())
    self_call("c4.full", 2, 16384, reverse=True)
    kvc_call(2, 16384, 4096)
    self_call("c5.self", 4, 4096, fp32_p=True)
    return calls


def sdpa_variants(q, k, v, mask):
    from torch.nn.attention import SDPBackend, sdpa_kernel
    out = {}
    for name, be in (("sdpa_flash", SDPBackend.FLASH_ATTENTION), ("sdpa_efficient", SDPBackend.EFFICIENT_ATTENTION),
                     ("sdpa_cudnn", SDPBackend.CUDNN_ATTENTION)):
        def fn(be=be):
            with sdpa_kernel(be):
                F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        try:
            fn()
            torch.cuda.synchronize()
        except RuntimeError:                                   # backend rejects head_dim 72, the strides or the mask
            continue
        out[name] = fn
    return out


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
    ap.add_argument("--seconds", type=float, default=1.0, help="timed launches per variant and call, in seconds (over all rounds)")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds over the variants; the median round is reported")
    ap.add_argument("--no-sdpa", action="store_true", help="time the library call only")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_attn.py measures on a GPU"
    from pixart_sigma_b200 import lib

    rows = []
    for name, (desc, flop, ours, sd) in make_calls(lib).items():
        variants = {"ours": ours}
        if not args.no_sdpa:
            variants.update(sdpa_variants(*sd))
        iters = {}
        for v, fn in variants.items():                         # warm-up, then size each window from a short timing
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            iters[v] = max(3, int(args.seconds / args.rounds / (time_window(fn, 3) * 1e-3)))
        times = {v: [] for v in variants}
        for _ in range(args.rounds):
            for v, fn in variants.items():
                times[v].append(time_window(fn, iters[v]))
        floor_ms = flop / (PEAK_TFLOPS * 1e12) * 1e3
        row = {"call": name, "shape": desc, "gflop": round(flop / 1e9, 2), "floor_ms": round(floor_ms, 4)}
        for v in variants:
            ms = sorted(times[v])[len(times[v]) // 2]
            row[v] = {"ms": round(ms, 4), "tflops": round(flop / (ms * 1e-3) / 1e12, 1), "share_of_floor": round(floor_ms / ms, 3),
                      "spread_ms": round(max(times[v]) - min(times[v]), 4)}
        rows.append(row)
        print(f"{name:9s} {desc} | floor {floor_ms:.3f} ms | " +
              " | ".join(f"{v} {row[v]['ms']:.3f} ms {row[v]['tflops']:.0f} TF/s ({row[v]['share_of_floor']:.0%})" for v in variants),
              file=sys.stderr)
    print(json.dumps({"workload": "head_dim-72 attention forward calls of c3 / c4 / c5", "calls": rows, "gpu": card()}))


if __name__ == "__main__":
    main()
