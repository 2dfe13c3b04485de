"""Text-to-image pipeline benchmark: prints one JSON line.

4 prompts at 1024 px through `pixart_sigma_b200.pipeline` with random-weight PixArt-Sigma XL/2 (28 blocks), T5-v1.1-XXL
(24 layers, d_model 4096) and SDXL-VAE, at inference.py's defaults (cfg 4.5, bs 4): DPM-Solver++ 20 steps and SA-Solver 25.
Reported per sampler, eager and with `cuda_graph=True` (which captures the loop on every call: the captured tensors are
per call), the whole generation from the prompt strings to uint8 pixels on the host, and for one eager run the stages:
tokenize + H2D, T5, sampling, decode (VAE up to conv_norm_out + SiLU), u8 + D2H (`pxa_vae_out_u8` and the copy).  Then
`pxa_vae_out_u8` alone against `F.conv2d` + the torch arithmetic of torchvision's save_image on the same 4 x 1024^2 input.
Times are wall clock around work that ends in a device synchronise (CUDA events for the kernel comparison), medians of
--reps runs after one warm-up.  Random weights: the timing does not depend on the values.  Writes nothing.
    python bench_pipeline.py [--reps 3]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def _random_(module, device, seed):
    """Give every parameter of a meta-device module random bf16 values on `device` (N(0, 1/fan_in); norms 1 + 0.1 N)."""
    g = torch.Generator(device=device).manual_seed(seed)
    for name, p in list(module.named_parameters()):
        if p.dim() > 1:
            v = torch.randn(p.shape, generator=g, device=device) * (p[0].numel() ** -0.5)
        elif "norm" in name and name.endswith("weight"):
            v = 1 + 0.1 * torch.randn(p.shape, generator=g, device=device)
        else:
            v = 0.1 * torch.randn(p.shape, generator=g, device=device)
        owner = module.get_submodule(name.rsplit(".", 1)[0]) if "." in name else module
        setattr(owner, name.rsplit(".", 1)[-1], torch.nn.Parameter(v.to(torch.bfloat16), requires_grad=False))
    return module.eval()


def _sync_time(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_pipeline.py needs a GPU"
    from transformers import T5Tokenizer
    from oracle.gen_golden_pipeline import write_tokenizer
    from pixart_sigma_b200 import lib, pipeline
    from pixart_sigma_b200.t5 import T5EncoderModel
    from pixart_sigma_b200.vae import AutoencoderKL
    dev = torch.device("cuda")
    torch.set_grad_enabled(False)
    with tempfile.TemporaryDirectory() as tmp:
        write_tokenizer(tmp)
        tok = T5Tokenizer.from_pretrained(tmp, subfolder="tokenizer")
    model = pipeline.build_transformer("sigma", 1024, dev).to(torch.bfloat16).eval()
    with torch.device("meta"):
        enc, vae = T5EncoderModel(), AutoencoderKL()
    enc, vae = _random_(enc, dev, 1), _random_(vae, dev, 2)
    enc.encoder.embed_tokens = enc.shared
    pipe = pipeline.PixArtPipeline(model, tok, enc, vae, "sigma", 1024)
    prompts = ["a lighthouse on a cliff at dusk, oil painting", "an astronaut riding a horse on the moon",
               "close-up portrait of an old fisherman, dramatic light", "a bowl of ramen, studio photo"]
    res = dict(workload="pipeline_1024_4prompts", gpu=_gpu_info(), reps=args.reps)

    def gen(algo, graph):
        return pipe.generate(prompts, sampling_algo=algo, bs=4, seed=0, cuda_graph=graph)["images"].cpu()

    for algo, key in (("dpm-solver", "dpm20"), ("sa-solver", "sa25")):
        for graph in (False, True):
            gen(algo, graph)
            ts = [_sync_time(lambda: gen(algo, graph))[0] for _ in range(args.reps)]
            res[f"{key}_{'graphed' if graph else 'eager'}_s"] = round(statistics.median(ts), 4)

    # stages of one eager DPM-Solver++ run
    st = {}
    st["tokenize_h2d"], (ids, mask) = _sync_time(lambda: pipe.tokenize(prompts))
    st["t5"], _ = _sync_time(lambda: enc(ids, attention_mask=mask))
    t_enc_and_sample, lat = _sync_time(lambda: pipe._sample(prompts, "dpm-solver", 20, 4.5, 128, 128, False, None, None))
    t_enc, _ = _sync_time(lambda: pipe.encode(prompts))
    st["sampling"] = t_enc_and_sample - t_enc
    dec = vae.decoder

    def trunk():
        z = F.conv2d((lat / vae.config.scaling_factor).to(torch.bfloat16), vae.post_quant_conv.weight, vae.post_quant_conv.bias)
        x = dec._trunk(z).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)
        n = dec.conv_norm_out
        return lib.groupnorm_silu_nhwc(x, n.weight, n.bias, torch.empty_like(x), groups=n.num_groups, eps=n.eps, silu=True)
    st["decode"], h = _sync_time(trunk)
    w_packed = dec.conv_out.weight.permute(0, 2, 3, 1).contiguous()
    bias = dec.conv_out.bias.float()
    u8 = torch.empty(*h.shape[:3], 3, dtype=torch.uint8, device=dev)
    st["u8_d2h"], _ = _sync_time(lambda: lib.vae_out_u8(h, w_packed, bias, u8).cpu())
    res["stages_dpm20_eager_s"] = {k: round(v, 4) for k, v in st.items()}

    # the output head alone: pxa_vae_out_u8 vs F.conv2d + save_image's arithmetic (torch)
    def torch_head():
        y = F.conv2d(h.permute(0, 3, 1, 2), dec.conv_out.weight, dec.conv_out.bias, padding=1).float()
        return y.clamp(-1, 1).sub(-1).div(2).mul(255).add(0.5).clamp(0, 255).to(torch.uint8)

    def ev_time(fn, n=20):
        fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n
    res["vae_out_u8_ms"] = round(ev_time(lambda: lib.vae_out_u8(h, w_packed, bias, u8)), 4)
    res["torch_conv_out_save_image_ms"] = round(ev_time(torch_head), 4)
    ref = torch_head().permute(0, 2, 3, 1)
    res["u8_max_abs_diff_vs_torch"] = int((u8.int() - ref.int()).abs().max())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
