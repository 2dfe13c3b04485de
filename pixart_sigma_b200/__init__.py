"""pixart_sigma_b200 -- H100-native (sm_90a) PixArt-Sigma DiT denoiser hot path.

Only what the path `PixArtMS.forward -> 28 x PixArtMSBlock.forward` needs:
  csrc/      hand-written CUDA (wgmma / TMA / mbarrier) behind the C-ABI of include/pixart_sm100.h
  lib.py     ctypes binding of libpixart_sm100.so
  model.py   host-side mirror of the reference model API (same names, ctor, state_dict layout)
  sampler.py DPM-Solver++ loop around the path (mirror of the reference's `diffusion.DPMS`), fused step kernel + CUDA graph
  sa_sampler.py  SA-Solver loop (mirror of the reference's `diffusion.SASolverSampler`), fused predictor-corrector step
             kernel + CUDA graph
  iddpm.py   IDDPM ancestral loop (mirror of the reference's `diffusion.IDDPM`), fused CFG-mix + ancestral step kernel + CUDA
             graph on CUDA latents, the torch restatement on CPU
  lcm.py     LCM: the few-step sampler (mirror of the reference's `LCMScheduler` loop) and consistency distillation with a
             fused flat EMA update
  dmd.py     DMD: distribution-matching distillation to a one-step generator (fused loss kernel) and one-step sampling
  lora.py    LoRA and DoRA adapters in peft's directory format, merged into the weights for sampling
  autograd.py / training.py  training path: the block's ops as autograd Functions over forward + backward kernels, IDDPM loss
  parallel.py  batch-sharded inference replicas; bucketed gradient all-reduce for data-parallel training
  vae.py / t5.py  the callers either side of the path on the same kernels: SDXL-VAE (diffusers' AutoencoderKL layout) and the
             T5-v1.1-XXL caption encoder (transformers' T5EncoderModel layout)
  pipeline.py / generate.py  text to image on these modules (the reference's scripts/inference.py flow) and its CLI
  build.py   in-tree nvcc build
"""
from .model import (MODELS, PixArt, PixArt_XL_2, PixArtBlock, PixArtMS, PixArtMS_XL_2, PixArtMSBlock,  # noqa: F401
                    build_model, install_into_reference, set_grad_checkpoint)
from .dmd import DMDDistiller, DMDSampler, ddpm_alphas_cumprod, null_caption  # noqa: F401
from .lora import (inject_dora, inject_lora, load_adapter, load_dora_adapter, merge_lora, save_adapter,  # noqa: F401
                   unmerge_lora)
from .lcm import LCMDistiller, LCMSampler, LCMScheduler  # noqa: F401
from .sa_sampler import SASolverSampler  # noqa: F401
from .sampler import DPMS, DPMSolverPP  # noqa: F401

__version__ = "0.1.0"
