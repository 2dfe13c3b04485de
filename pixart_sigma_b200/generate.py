"""Command line text-to-image generation: `python -m pixart_sigma_b200.generate --txt_file prompts.txt ...`.

Takes scripts/inference.py's arguments (`--txt_file --image_size --version --model_path --pipeline_load_from --bs --cfg_scale
--sampling_algo --seed --step --sdvae`) plus `--height/--width` (explicit size, multiples of 16 px; there is no aspect-ratio
binning), `--out_dir` and `--cuda_graph`, and writes one `"{prompt[:100]}.jpg"` per prompt, encoded by PIL with its default
settings as torchvision's save_image does.
"""
from __future__ import annotations

import argparse
import os
from typing import List, Optional

from .pipeline import DEFAULT_STEPS, MAX_LENGTH


def get_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(prog="python -m pixart_sigma_b200.generate", description=__doc__.split("\n")[0])
    p.add_argument("--image_size", default=1024, type=int)
    p.add_argument("--version", default="sigma", type=str, choices=sorted(MAX_LENGTH))
    p.add_argument("--pipeline_load_from", default="output/pretrained_models/pixart_sigma_sdxlvae_T5_diffusers", type=str,
                   help="diffusers pipeline directory with tokenizer/, text_encoder/ and vae/")
    p.add_argument("--txt_file", default="asset/samples.txt", type=str, help="one prompt per line")
    p.add_argument("--model_path", default="output/pretrained_models/PixArt-XL-2-1024x1024.pth", type=str,
                   help="reference .pth checkpoint, or diffusers transformer weights (.safetensors file or directory)")
    p.add_argument("--sdvae", action="store_true", help="SD-VAE from output/pretrained_models/sd-vae-ft-ema")
    p.add_argument("--bs", default=1, type=int)
    p.add_argument("--cfg_scale", default=4.5, type=float)
    p.add_argument("--sampling_algo", default="dpm-solver", type=str, choices=list(DEFAULT_STEPS))
    p.add_argument("--seed", default=0, type=int)
    p.add_argument("--step", default=-1, type=int, help="-1: 100 (iddpm) / 20 (dpm-solver) / 25 (sa-solver)")
    p.add_argument("--height", default=None, type=int, help="image height in px (default: image_size)")
    p.add_argument("--width", default=None, type=int, help="image width in px (default: image_size)")
    p.add_argument("--out_dir", default="output/samples", type=str)
    p.add_argument("--cuda_graph", action="store_true", help="run each sampling loop as one CUDA graph")
    return p


def read_prompts(path: str) -> List[str]:
    with open(path) as f:
        return [line.strip() for line in f.readlines()]


def save_images(images_u8, prompts: List[str], out_dir: str) -> List[str]:
    """Write uint8 (n, H, W, 3) host images as `{prompt[:100]}.jpg` with PIL's defaults (torchvision's save_image)."""
    from PIL import Image
    os.makedirs(out_dir, exist_ok=True)
    paths = []
    for img, prompt in zip(images_u8.numpy(), prompts):
        path = os.path.join(out_dir, f"{prompt[:100]}.jpg")
        Image.fromarray(img).save(path)
        paths.append(path)
    return paths


def main(argv: Optional[List[str]] = None, pipeline=None) -> List[str]:
    """Parse `argv`, generate and save; `pipeline` replaces the one loaded from the paths.  Returns the written paths."""
    args = get_parser().parse_args(argv)
    from .pipeline import PixArtPipeline
    if pipeline is None:
        pipeline = PixArtPipeline.from_pretrained(args.model_path, args.pipeline_load_from, version=args.version,
                                                  image_size=args.image_size, sdvae=args.sdvae)
    prompts = read_prompts(args.txt_file)
    res = pipeline.generate(prompts, sampling_algo=args.sampling_algo, steps=args.step, cfg_scale=args.cfg_scale,
                            seed=args.seed, bs=args.bs, height=args.height, width=args.width, cuda_graph=args.cuda_graph)
    paths = save_images(res["images"].cpu(), res["prompts"], args.out_dir)
    for p in paths:
        print("Saving path:", p)
    return paths


if __name__ == "__main__":
    main()
