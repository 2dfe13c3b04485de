"""Training step around the denoiser (SURVEY.md 8a rows 17, 18, 20; BASELINE configs[4]).

`IDDPMLoss` restates the loss the reference trains with -- `IDDPM(str(1000), learn_sigma=True, pred_sigma=True,
snr=False)` (`train_scripts/train.py:410`, `diffusion/iddpm.py:10-53`) -> `SpacedDiffusion.training_losses`
(`diffusion/model/gaussian_diffusion.py:744-855`): q_sample, epsilon MSE, and the learned-range variational-bound term
computed on a detached mean (`:805-819`, `_vb_terms_bpd :711-742`).  It is host glue on (n, 4, h, w) latents (a few
elementwise torch ops, no kernels of ours; SURVEY.md 8a row 18 keeps the outer loops in PyTorch); the fp64 schedule
tables are built once.  Pinned against the unmodified reference by `tests/golden/train_*.pt`.

`train_step` = loss forward + backward through the sm_90a kernel ops (`autograd.py`), optionally with the bucketed
gradient all-reduce of `parallel.GradBucketReducer` overlapping the backward (row 20, `train.py:180-197`).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch


class IDDPMLoss:
    """`IDDPM('1000', noise_schedule='linear', learn_sigma=True, pred_sigma=True, snr=False)` training loss."""

    def __init__(self, diffusion_steps: int = 1000):
        scale = 1000 / diffusion_steps                                        # gaussian_diffusion.py:107-116
        betas = np.linspace(scale * 0.0001, scale * 0.02, diffusion_steps, dtype=np.float64)
        alphas = 1.0 - betas
        ac = np.cumprod(alphas, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        self.num_timesteps = diffusion_steps
        post_var = betas * (1.0 - ac_prev) / (1.0 - ac)                       # :214-227
        self.tab = {
            "sqrt_ac": np.sqrt(ac), "sqrt_1mac": np.sqrt(1.0 - ac),
            "sqrt_recip_ac": np.sqrt(1.0 / ac), "sqrt_recipm1_ac": np.sqrt(1.0 / ac - 1),
            "post_logvar": np.log(np.append(post_var[1], post_var[1:])),
            "post_c1": betas * np.sqrt(ac_prev) / (1.0 - ac), "post_c2": (1.0 - ac_prev) * np.sqrt(alphas) / (1.0 - ac),
            "log_betas": np.log(betas),
        }
        self._dev: Dict[str, torch.Tensor] = {}

    def _x(self, name: str, t: torch.Tensor) -> torch.Tensor:
        """_extract_into_tensor (:1029-1041): fp64 table -> indexed -> fp32, broadcast over (n, 1, 1, 1)."""
        key = f"{name}@{t.device}"
        if key not in self._dev:
            self._dev[key] = torch.from_numpy(self.tab[name]).to(t.device)
        return self._dev[key][t].float()[:, None, None, None]

    def q_sample(self, x_start, t, noise):                                   # :243-256
        return self._x("sqrt_ac", t) * x_start + self._x("sqrt_1mac", t) * noise

    def _vb(self, eps_detached, var_values, x_start, x_t, t):
        """_vb_terms_bpd (:711-742) with p_mean_variance's LEARNED_RANGE branch (:311-319), clip_denoised=False."""
        true_mean = self._x("post_c1", t) * x_start + self._x("post_c2", t) * x_t
        true_logvar = self._x("post_logvar", t)
        frac = (var_values + 1) / 2
        logvar = frac * self._x("log_betas", t) + (1 - frac) * true_logvar
        pred_x0 = self._x("sqrt_recip_ac", t) * x_t - self._x("sqrt_recipm1_ac", t) * eps_detached
        mean = self._x("post_c1", t) * pred_x0 + self._x("post_c2", t) * x_t
        kl = 0.5 * (-1.0 + logvar - true_logvar + torch.exp(true_logvar - logvar) + (true_mean - mean) ** 2 * torch.exp(-logvar))
        kl = kl.flatten(1).mean(1) / math.log(2.0)
        # decoder NLL at t == 0: discretized Gaussian log-likelihood (diffusion_utils.py:60-88)
        cdf = lambda v: 0.5 * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (v + 0.044715 * v ** 3)))
        centered, inv_std = x_start - mean, torch.exp(-0.5 * logvar)
        cdf_plus, cdf_min = cdf(inv_std * (centered + 1.0 / 255.0)), cdf(inv_std * (centered - 1.0 / 255.0))
        log_probs = torch.where(x_start < -0.999, torch.log(cdf_plus.clamp(min=1e-12)),
                                torch.where(x_start > 0.999, torch.log((1.0 - cdf_min).clamp(min=1e-12)),
                                            torch.log((cdf_plus - cdf_min).clamp(min=1e-12))))
        nll = -log_probs.flatten(1).mean(1) / math.log(2.0)
        return torch.where(t == 0, nll, kl)

    def training_losses(self, model, x_start, timestep, model_kwargs: Optional[dict] = None, noise=None) -> Dict[str, torch.Tensor]:
        """Same signature and result keys ('mse', 'vb', 'loss', each (n,)) as gaussian_diffusion.py:744."""
        t = timestep
        if noise is None:
            noise = torch.randn_like(x_start)
        x_t = self.q_sample(x_start, t, noise)
        out = model(x_t, timestep=t, **(model_kwargs or {}))          # keyword, as respace.py:134 calls it
        out = out.float()
        C = x_t.shape[1]
        assert out.shape == (x_t.shape[0], 2 * C, *x_t.shape[2:])
        eps, var_values = torch.split(out, C, dim=1)
        terms = {"vb": self._vb(eps.detach(), var_values, x_start, x_t, t),
                 "mse": ((noise - eps) ** 2).flatten(1).mean(1)}
        terms["loss"] = terms["mse"] + terms["vb"]
        return terms


class DDPMEpsLoss:
    """The objective of `train_scripts/train_pixart_lora_hf.py`: noise added by diffusers' `DDPMScheduler.add_noise` on its
    float32 alphas_cumprod (`dmd.ddpm_alphas_cumprod`), model_pred = the first half of the output channels (the epsilon
    prediction; the learned variance is not trained), and the MSE against the noise.  `training_losses` has IDDPMLoss's
    contract; its 'loss' is the per-sample mean, so that loss.mean() is the script's `F.mse_loss(..., reduction="mean")`.
    For LoRA, build the model with class_dropout_prob=0 (the script's diffusers transformer drops no captions) and keep the
    adapter unmerged while training."""

    def __init__(self, num_train_timesteps: int = 1000, snr_gamma: Optional[float] = None, prediction_type: str = "epsilon"):
        from .dmd import ddpm_alphas_cumprod
        if snr_gamma is not None:
            raise NotImplementedError("snr_gamma loss weighting is not supported")
        if prediction_type != "epsilon":
            raise NotImplementedError(f"prediction_type={prediction_type!r} is not supported (only 'epsilon')")
        self.num_timesteps = num_train_timesteps
        self.alphas_cumprod = ddpm_alphas_cumprod(num_train_timesteps)
        self._dev: Dict[str, torch.Tensor] = {}

    def training_losses(self, model, x_start, timestep, model_kwargs: Optional[dict] = None, noise=None) -> Dict[str, torch.Tensor]:
        from .dmd import ddpm_add_noise
        if noise is None:
            noise = torch.randn_like(x_start)
        key = str(x_start.device)
        if key not in self._dev:
            self._dev[key] = self.alphas_cumprod.to(x_start.device)
        x_t = ddpm_add_noise(self._dev[key], x_start, noise, timestep)
        out = model(x_t, timestep=timestep, **(model_kwargs or {}))
        pred = out.chunk(2, 1)[0].float()
        mse = ((pred - noise.float()) ** 2).flatten(1).mean(1)
        return {"mse": mse, "loss": mse}


def train_step(model, loss_fn: IDDPMLoss, x_start, timestep, y, mask, data_info=None, noise=None, reducer=None,
               loss_scale: float = 1.0, refresh_shadows: bool = True) -> torch.Tensor:
    """One fwd + bwd of `train_scripts/train.py:186-197` (the optimizer step stays the caller's): returns the mean loss
    (detached).  With `reducer` (parallel.GradBucketReducer) the gradient all-reduce runs bucket by bucket behind the
    backward and is complete when this returns.  `refresh_shadows`: re-derive the cached bf16 weight shadows from the
    parameters at the start of the step, which makes in-place `.data` updates between steps safe."""
    if refresh_shadows:
        from . import autograd as ag
        ag.refresh_shadows(model)           # `.data` writes (fused / ZeRO optimizers, EMA copies) do not bump `_version`
    if reducer is not None:
        reducer.start()
    terms = loss_fn.training_losses(model, x_start, timestep, dict(y=y, mask=mask, data_info=data_info), noise=noise)
    loss = terms["loss"].mean()
    (loss * loss_scale).backward()
    if reducer is not None:
        reducer.finish()
    return loss.detach()


class GraphedTrainStep:
    """One training step (gradient zeroing + loss forward + backward through the kernels) captured as ONE CUDA graph.

    The eager step issues ~10 k kernel launches through Python / autograd, whose host cost competes with the time the GPU needs
    to run them, so the step is captured once with static
    input buffers and replayed; the library never allocates or synchronises and autograd's backward runs on the capture
    stream, so fwd + bwd capture as they are.  Every replay first refreshes the bf16 weight shadows IN PLACE from the
    (optimizer-updated) fp32 parameters (`autograd.refresh_shadows`, part of the graph), so an optimizer step between
    replays is seen.  The gradient all-reduce: by default it stays outside the graph -- `reducer.finish()` reduces the flat
    buckets after the replay (exposed, no overlap with the backward); with `capture_collectives=True` the bucket all-reduces
    are captured too, on NCCL's stream, forked from the backward where each bucket completes and joined at the end of the
    graph, so replays overlap them with the rest of the backward exactly like the eager path does.

    Fixed shapes only (one graph per batch geometry); activation checkpointing is captured as well (the recomputation is
    just more kernels on the stream; torch's RNG-state stashing, which reads the device, is disabled).
    """

    def __init__(self, model, loss_fn: IDDPMLoss, reducer, example, warmup: int = 2, capture_collectives: bool = False):
        from . import autograd as ag
        self.model, self.loss_fn, self.reducer = model, loss_fn, reducer
        self.captured = bool(capture_collectives) and reducer.world > 1
        reducer.overlap = self.captured              # False: collectives stay outside the graph
        dev = next(model.parameters()).device
        self.static = [None if v is None else torch.empty_like(v, device=dev) for v in example]
        self._copy_in(example)
        x0, t, y, mask, noise = self.static

        def step():
            ag.refresh_shadows(model)
            reducer.zero_grad()
            if self.captured:
                reducer.start()
            terms = loss_fn.training_losses(model, x0, t, dict(y=y, mask=mask, data_info=None), noise=noise)
            loss = terms["loss"].mean()
            loss.backward()
            if self.captured:
                reducer.finish()
            return loss.detach()

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(warmup):                       # eager: allocator warm-up, shadows and caches created
                step()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        # thread_local: NCCL's watchdog thread may query events while this thread captures
        with torch.cuda.graph(self.graph, capture_error_mode="thread_local" if self.captured else "global"):
            self.loss = step()

    def _copy_in(self, batch):
        for dst, src in zip(self.static, batch):
            if dst is not None:
                dst.copy_(src, non_blocking=True)

    def __call__(self, x_start, timestep, y, mask, noise) -> torch.Tensor:
        self._copy_in((x_start, timestep, y, mask, noise))
        if self.captured:
            self.reducer.check_views()
            self.graph.replay()
            return self.loss
        self.reducer.start()
        self.graph.replay()
        if self.reducer.world > 1:
            self.reducer.finish()
        return self.loss
