"""Text-to-image generation on the native modules: prompts -> tokens -> T5 -> sampling loop -> VAE -> uint8 pixels.

This is the `visualize()` flow of the reference's scripts/inference.py (lines 53-143, set-up 146-224) without the reference
or diffusers: the transformer is `model.PixArtMS` / `model.PixArt`, the caption encoder `t5.T5EncoderModel`, the samplers
`sampler.DPMS`, `sa_sampler.SASolverSampler` and `iddpm.IDDPM`, the autoencoder `vae.AutoencoderKL`, whose output head
writes image bytes directly (`decode_to_uint8`, kernel `pxa_vae_out_u8`).  The script's behaviour is kept, quirks included:
the seed set-up (`set_env`), prompt cleaning, both CFG halves masked with the conditional prompt's mask, SA-Solver at
S = 25 whatever the step count, and the order of every random draw, so that a seed draws the numbers the script would draw
on the same GPU.  Deliberate deviations: a batch of one prompt works (the script's bs == 1 branch raises IndexError),
there is no aspect-ratio binning (explicit `height` / `width` instead), and the VAE runs in bf16 (the script: fp16).

Between the token upload and the caller's copy of the pixels to the host nothing waits for the device: the tokens and
the masks go up through pinned memory, and every later step is a device operation.
"""
from __future__ import annotations

import json
import os
from typing import Dict, List, Optional, Sequence

import torch

from . import convert
from .iddpm import IDDPM
from .model import PixArt, PixArtMS
from .sa_sampler import SASolverSampler
from .sampler import DPMS
from .t5 import T5_V1_1_XXL, T5EncoderModel
from .vae import SDXL_VAE_CONFIG, AutoencoderKL

MAX_LENGTH = {"alpha": 120, "sigma": 300}                       # inference.py:156
DEFAULT_STEPS = {"iddpm": 100, "dpm-solver": 20, "sa-solver": 25}  # inference.py:159
SAMPLERS = tuple(DEFAULT_STEPS)
SA_SOLVER_STEPS = 25                                            # inference.py:125 hard-codes S=25


def clean_prompt(prompt: str) -> str:
    """`prepare_prompt_ar(prompt, ...)[0].strip()`: the text before `--aspect_ratio`, then `--ar`, then `--hw`."""
    return prompt.split("--aspect_ratio")[0].split("--ar")[0].split("--hw")[0].strip()


def get_chunks(items: Sequence, n: int):
    for i in range(0, len(items), n):
        yield items[i:i + n]


def transformer_config(version: str = "sigma", image_size: int = 1024) -> dict:
    """Constructor of inference.py:154-178: `name` is "PixArtMS_XL_2" or "PixArt_XL_2", `kwargs` its arguments."""
    if version not in MAX_LENGTH:
        raise ValueError(f"version must be one of {sorted(MAX_LENGTH)}, got {version!r}")
    kwargs = dict(input_size=image_size // 8, pe_interpolation=image_size / 512, model_max_length=MAX_LENGTH[version])
    if image_size in (512, 1024, 2048) or version == "sigma":
        return dict(name="PixArtMS_XL_2", kwargs=dict(kwargs, micro_condition=version == "alpha" and image_size == 1024))
    return dict(name="PixArt_XL_2", kwargs=kwargs)


def build_transformer(version: str = "sigma", image_size: int = 1024, device="cuda", **overrides) -> PixArtMS:
    """The XL/2 model of `transformer_config` (fp32, initialised) on `device`; `overrides` replace architecture arguments
    (depth, hidden_size, caption_channels, ...) for small test models."""
    spec = transformer_config(version, image_size)
    arch = dict(depth=28, hidden_size=1152, patch_size=2, num_heads=16)
    arch.update(overrides)
    cls = PixArtMS if spec["name"] == "PixArtMS_XL_2" else PixArt
    with torch.device(device):
        return cls(**arch, **spec["kwargs"])


def read_transformer_state_dict(model_path: str, micro_condition: bool = False) -> Dict[str, torch.Tensor]:
    """A reference checkpoint `.pth` (`{'state_dict': ...}`, inference.py:181-184, `pos_embed` dropped), or a diffusers
    transformer (`.safetensors` file, or a directory with `transformer/diffusion_pytorch_model.safetensors` or
    `diffusion_pytorch_model.safetensors`) re-keyed by `convert.from_diffusers`."""
    path = model_path
    if os.path.isdir(path):
        for cand in ("transformer/diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.safetensors"):
            if os.path.isfile(os.path.join(path, cand)):
                path = os.path.join(path, cand)
                break
        else:
            raise FileNotFoundError(f"no diffusers transformer weights under {model_path}")
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        dsd = load_file(path)
        qk_norm = any(".attn1.q_norm." in k for k in dsd)
        return convert.from_diffusers(dsd, micro_condition=micro_condition, qk_norm=qk_norm)
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    if not isinstance(ckpt, dict) or "state_dict" not in ckpt:
        raise ValueError(f"{model_path}: expected a checkpoint dict with a 'state_dict' entry")
    sd = dict(ckpt["state_dict"])
    sd.pop("pos_embed", None)
    return sd


def load_transformer(model_path: str, version: str = "sigma", image_size: int = 1024, device="cuda", **overrides):
    """Build as inference.py does, load with strict=False, cast to bf16, eval().  Returns (model, missing, unexpected)."""
    m = build_transformer(version, image_size, device, **overrides)
    sd = read_transformer_state_dict(model_path, micro_condition=m.micro_conditioning)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    return m.to(torch.bfloat16).eval(), missing, unexpected


def _safetensors_files(folder: str, stem: str) -> List[str]:
    """`{stem}.safetensors`, or the shards named by `{stem}.safetensors.index.json`."""
    index = os.path.join(folder, stem + ".safetensors.index.json")
    if os.path.isfile(index):
        with open(index) as f:
            shards = sorted(set(json.load(f)["weight_map"].values()))
        return [os.path.join(folder, s) for s in shards]
    single = os.path.join(folder, stem + ".safetensors")
    if os.path.isfile(single):
        return [single]
    raise FileNotFoundError(f"no {stem}.safetensors or {stem}.safetensors.index.json in {folder}")


def _load_bf16(module: torch.nn.Module, files: Sequence[str], device, allow_missing=()) -> torch.nn.Module:
    """Fill a module built on the meta device from safetensors files, one tensor at a time: each is cast to bf16 on the
    host and then copied to `device`, so no fp32 copy of the weights ever reaches the GPU."""
    from safetensors import safe_open
    sd = {}
    for fn in files:
        with safe_open(fn, framework="pt", device="cpu") as f:
            for k in f.keys():
                sd[k] = f.get_tensor(k).to(torch.bfloat16).to(device)
    missing, unexpected = module.load_state_dict(sd, strict=False, assign=True)
    missing = [k for k in missing if k not in allow_missing]
    if missing or unexpected:
        raise RuntimeError(f"{type(module).__name__}: checkpoint layout mismatch: missing {missing}, unexpected {unexpected}")
    return module.eval()


def load_text_encoder(pipeline_load_from: str, device="cuda"):
    """(tokenizer, T5EncoderModel) from a diffusers pipeline directory: `tokenizer/` for transformers' T5Tokenizer,
    `text_encoder/config.json` and the single-file or sharded `model.safetensors` for the native encoder (bf16, `device`)."""
    from transformers import T5Tokenizer
    tokenizer = T5Tokenizer.from_pretrained(pipeline_load_from, subfolder="tokenizer")
    folder = os.path.join(pipeline_load_from, "text_encoder")
    with open(os.path.join(folder, "config.json")) as f:
        hf = json.load(f)
    cfg = {k: hf[k] for k in T5_V1_1_XXL if k in hf}
    with torch.device("meta"):
        enc = T5EncoderModel(cfg)
    # `encoder.embed_tokens` is the `shared` module itself: a file may leave out its key
    return tokenizer, _load_bf16(enc, _safetensors_files(folder, "model"), device, allow_missing=("encoder.embed_tokens.weight",))


def load_vae(folder: str, device="cuda") -> AutoencoderKL:
    """The native AutoencoderKL from a diffusers `vae/` directory (`config.json`: block widths, scaling_factor, ...;
    `diffusion_pytorch_model.safetensors`): the SDXL-VAE of the Sigma pipeline, or the SD-VAE of `--sdvae`."""
    with open(os.path.join(folder, "config.json")) as f:
        hf = json.load(f)
    cfg = dict(SDXL_VAE_CONFIG)
    cfg.update({k: (tuple(hf[k]) if k == "block_out_channels" else hf[k]) for k in SDXL_VAE_CONFIG if k in hf})
    with torch.device("meta"):
        vae = AutoencoderKL(cfg)
    return _load_bf16(vae, _safetensors_files(folder, "diffusion_pytorch_model"), device)


def _upload(t: torch.Tensor, device) -> torch.Tensor:
    """Host tensor -> device without waiting for the copy (pinned staging buffer)."""
    return t.pin_memory().to(device, non_blocking=True)


class PixArtPipeline:
    """The script's generation loop on native modules.  `generate` returns uint8 images on the device."""

    def __init__(self, transformer: PixArtMS, tokenizer, text_encoder: T5EncoderModel, vae: AutoencoderKL,
                 version: str = "sigma", image_size: int = 1024):
        if version not in MAX_LENGTH:
            raise ValueError(f"version must be one of {sorted(MAX_LENGTH)}, got {version!r}")
        self.transformer, self.tokenizer, self.text_encoder, self.vae = transformer, tokenizer, text_encoder, vae
        self.version, self.image_size = version, int(image_size)
        self.max_length = MAX_LENGTH[version]
        self.device = transformer.blocks[0].attn.qkv.weight.device
        if self.device.type != "cuda":
            raise RuntimeError("PixArtPipeline runs on the sm_90a kernels only: the transformer must be on a CUDA device")
        self._null = None

    @classmethod
    def from_pretrained(cls, model_path: str, pipeline_load_from: str, version: str = "sigma", image_size: int = 1024,
                        sdvae: bool = False, device="cuda") -> "PixArtPipeline":
        """inference.py:164-202: the transformer from `model_path`; tokenizer, T5 and VAE from `pipeline_load_from`
        (`sdvae`: the SD-VAE at output/pretrained_models/sd-vae-ft-ema, as the script loads it)."""
        model = load_transformer(model_path, version, image_size, device)[0]
        vae = load_vae("output/pretrained_models/sd-vae-ft-ema" if sdvae else os.path.join(pipeline_load_from, "vae"), device)
        tokenizer, enc = load_text_encoder(pipeline_load_from, device)
        return cls(model, tokenizer, enc, vae, version, image_size)

    # ---- captions
    def tokenize(self, prompts: List[str]):
        """(input_ids, attention_mask) on the device, padded to max_length (120 / 300) and truncated."""
        tok = self.tokenizer(prompts, max_length=self.max_length, padding="max_length", truncation=True, return_tensors="pt")
        return _upload(tok.input_ids, self.device), _upload(tok.attention_mask, self.device)

    def encode(self, prompts: List[str]):
        """(caption embeddings (n, L, D) bf16, attention mask (n, L)) on the device."""
        ids, mask = self.tokenize(prompts)
        return self.text_encoder(ids, attention_mask=mask)[0], mask

    def null_embedding(self) -> torch.Tensor:
        """T5 of the empty caption (1, L, D), computed once (inference.py:201-202)."""
        if self._null is None:
            self._null = self.encode([""])[0]
        return self._null

    # ---- generation
    def set_seed(self, seed: int) -> None:
        """`set_env(seed)` of inference.py:47-51: seed every generator, then 30 CPU draws of (1, 4, S, S)."""
        torch.manual_seed(seed)
        for _ in range(30):
            torch.randn(1, 4, self.image_size, self.image_size)

    @torch.no_grad()
    def generate(self, prompts: Sequence[str], *, sampling_algo: str = "dpm-solver", steps: Optional[int] = None,
                 cfg_scale: float = 4.5, seed: Optional[int] = 0, bs: int = 1, height: Optional[int] = None,
                 width: Optional[int] = None, cuda_graph: bool = False, return_float: bool = False,
                 return_latents: bool = False, x_T: Optional[torch.Tensor] = None,
                 noise_draws: Optional[Sequence[Sequence[torch.Tensor]]] = None) -> dict:
        """Images for `prompts`, `bs` at a time, as inference.py's visualize() makes them.

        Returns a dict: `images` uint8 (n, H, W, 3) on the device (what save_image turns into a file, before the JPEG
        encoder), `prompts` the cleaned prompts, and on request `float` (n, 3, H, W) fp32 (the VAE output) and `latents`
        (n, 4, H/8, W/8) fp32 (the sampler output).  `seed=None` skips the seed set-up (the generators continue).
        Replay: `x_T` (n, 4, H/8, W/8) replaces the initial draws, `noise_draws[k]` the sampler's per-step draws of chunk k
        (IDDPM: one (2n_k, 4, h, w) per step; SA-Solver: the 25 draws after its discarded one; DPM-Solver++ draws none)."""
        if sampling_algo not in SAMPLERS:
            raise ValueError(f"sampling_algo must be one of {SAMPLERS}, got {sampling_algo!r}")
        if bs < 1:
            raise ValueError("bs must be >= 1")
        H, W = int(height or self.image_size), int(width or self.image_size)
        if H <= 0 or W <= 0 or H % 16 or W % 16:
            raise ValueError(f"height and width must be positive multiples of 16 px, got {H} x {W}")
        steps = DEFAULT_STEPS[sampling_algo] if steps is None or steps == -1 else int(steps)
        items = [clean_prompt(p) for p in prompts]
        if x_T is not None and tuple(x_T.shape) != (len(items), 4, H // 8, W // 8):
            raise ValueError(f"x_T must have shape {(len(items), 4, H // 8, W // 8)}")
        if seed is not None:
            self.set_seed(seed)
        images, floats, latents = [], [], []
        for k, chunk in enumerate(get_chunks(items, bs)):
            lo = k * bs
            z = None if x_T is None else x_T[lo:lo + len(chunk)].to(self.device, torch.float32)
            draws = None if noise_draws is None else noise_draws[k]
            samples = self._sample(list(chunk), sampling_algo, steps, cfg_scale, H // 8, W // 8, cuda_graph, z, draws)
            if return_latents:
                latents.append(samples)
            out = self.vae.decode_to_uint8(samples / self.vae.config.scaling_factor, return_float=return_float)
            if return_float:
                images.append(out[0])
                floats.append(out[1])
            else:
                images.append(out)
        res = dict(images=torch.cat(images), prompts=items)
        if return_float:
            res["float"] = torch.cat(floats)
        if return_latents:
            res["latents"] = torch.cat(latents)
        return res

    def _sample(self, prompts, algo, steps, cfg_scale, h, w, cuda_graph, z, draws) -> torch.Tensor:
        n, dev, m = len(prompts), self.device, self.transformer
        emb, mask = self.encode(prompts)
        caption_embs = emb[:, None]                                                    # (n, 1, L, D)
        null_y = self.null_embedding().repeat(n, 1, 1)[:, None]
        data_info = {"img_hw": torch.tensor([[8.0 * h, 8.0 * w]]).repeat(n, 1).pin_memory().to(dev, non_blocking=True),
                     "aspect_ratio": torch.ones(n, 1, device=dev)}
        if algo == "iddpm":
            if z is None:
                z = torch.randn(n, 4, h, w, device=dev)
            z = z.repeat(2, 1, 1, 1)
            kwargs = dict(y=torch.cat([caption_embs, null_y]), cfg_scale=cfg_scale, data_info=data_info, mask=mask)
            out = IDDPM(str(steps)).p_sample_loop(m.forward_with_cfg, z.shape, z, clip_denoised=False, model_kwargs=kwargs,
                                                   device=dev, noise_draws=draws, cuda_graph=cuda_graph)
            return out.chunk(2, dim=0)[0]
        kwargs = dict(data_info=data_info, mask=mask)
        if algo == "dpm-solver":
            if z is None:
                z = torch.randn(n, 4, h, w, device=dev)
            solver = DPMS(m.forward_with_dpmsolver, condition=caption_embs, uncondition=null_y, cfg_scale=cfg_scale,
                          model_kwargs=kwargs)
            return solver.sample(z, steps=steps, order=2, skip_type="time_uniform", method="multistep", cuda_graph=cuda_graph)
        sa = SASolverSampler(m.forward_with_dpmsolver, device=dev)
        return sa.sample(S=SA_SOLVER_STEPS, batch_size=n, shape=(4, h, w), eta=1, conditioning=caption_embs,
                         unconditional_conditioning=null_y, unconditional_guidance_scale=cfg_scale, model_kwargs=kwargs,
                         x_T=z, noise=draws, cuda_graph=cuda_graph)[0]
