"""DMD on the sm_90a kernels: distribution-matching distillation to a one-step generator, and one-step sampling.

Mirrors `train_scripts/train_pixart_dmd.py` with `use_dm`, no regression loss, `snr_gamma=None` and `noise_offset=0`, at the
settings of `scripts/run_pixart_dmd.py` (cfg 3, start_ts 999, one_step_maxt 999, `--use_ema`), and the sampling of
`app/app_pixart_dmd.py`:
  * `ddpm_alphas_cumprod` -- the float32 `alphas_cumprod` of diffusers' `DDPMScheduler` (linear betas 1e-4 .. 0.02), the
    table DMD uses throughout (not IDDPM's fp64 one).
  * `DMDSampler` -- one denoiser evaluation and `pxa_lcm_step` as x0-from-eps: `eps_to_mu` (scripts/DMD/transformer_train/
    generate.py:34-41) at t = 400 (the app's single `DDPMScheduler` step, whose arithmetic at prev_t < 0 is eps_to_mu; the
    variance it adds is clamped to about 1e-10 and left out) or at t = 999 (`generate_sample_1step`).  Optionally replayed
    from one CUDA graph.
  * `DMDDistiller` -- one training step (:484-687): the generator's one-step x0, the distribution-matching loss from one
    batch-2b forward of the frozen real model over [uncond ; cond] and the fake model's forward, both reduced by one
    `pxa_dmd_loss` sequence that writes the gradient with respect to the generator's output; then the fake model's
    denoising loss.  Both backward passes run into their reducers before the caller's optimizer steps, which is the
    reference's order: the fake step only reads the generator's detached output.  `update_ema()` is diffusers' `EMAModel.step`
    as one `pxa_ema_flat` launch.
  * `null_caption` -- the unconditional caption (the T5 embedding of "") from the native T5 encoder.
The caller keeps `optim.clip_grad_norm_` and `optim.FlatAdamW` as they are.  There is no CPU path.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Sequence, Tuple

import torch

from . import lib
from .lcm import FlatEMA, LCMScheduler, _ConsistencyLoss, _dup, _inference_copy, _upload
from .capture import CapturedLoops, step_input

__all__ = ["ddpm_alphas_cumprod", "ddpm_add_noise", "ema_decay", "dmd_draws", "null_caption", "DMDSampler", "DMDDistiller"]


def ddpm_alphas_cumprod(num_train_timesteps: int = 1000) -> torch.Tensor:
    """float32 cumprod(1 - linspace(1e-4, 0.02, T)), as diffusers' `DDPMScheduler` and `LCMScheduler` compute it."""
    return LCMScheduler(num_train_timesteps=num_train_timesteps).alphas_cumprod


def ddpm_add_noise(alphas_cumprod: torch.Tensor, x: torch.Tensor, noise: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    """`DDPMScheduler.add_noise` on a float32 alphas_cumprod table (on x's device): sqrt(a_t) x + sqrt(1 - a_t) noise."""
    a = alphas_cumprod[t]
    return (a ** 0.5).view(-1, 1, 1, 1) * x + ((1 - a) ** 0.5).view(-1, 1, 1, 1) * noise


def ema_decay(update: int, max_decay: float = 0.9999) -> float:
    """The decay of the `update`-th (1-based) `EMAModel.step` with the defaults `train_pixart_dmd.py:230` keeps
    (update_after_step 0, no warm-up, min_decay 0): 0 on the first update, then min((1 + s) / (10 + s), max_decay) with
    s = update - 1.  Restated from diffusers' `diffusers/training_utils.py` (`EMAModel.get_decay`); diffusers is not part of
    the reference tree, so the version is unpinned."""
    s = max(0, int(update) - 1)
    return 0.0 if s <= 0 else min((1 + s) / (10 + s), float(max_decay))


def dmd_draws(b: int, hw: Sequence[int], device, start_ts: int = 999, fix_noise_ts: Optional[int] = None):
    """The random inputs of one step in the reference's device-RNG order: init_noise (:484), noise and timesteps (:495, :507),
    noise_f and t_f (:628, :635).  Returns (init_noise, noise, t, noise_f, t_f)."""
    h, w = hw
    init_noise = torch.randn((b, 4, h, w), dtype=torch.float32, device=device)
    noise = torch.randn_like(init_noise)
    t = torch.randint(1, start_ts, (b,), device=device)
    if fix_noise_ts is not None:
        t = 0 * t + fix_noise_ts
    noise_f = torch.randn_like(init_noise)
    t_f = torch.randint(1, start_ts, (b,), device=device)
    if fix_noise_ts is not None:
        t_f = 0 * t_f + fix_noise_ts
    return init_noise, noise, t.long(), noise_f, t_f.long()


@torch.no_grad()
def null_caption(t5, max_length: int = 300) -> Tuple[torch.Tensor, torch.Tensor]:
    """(y (1, 1, L, d_model), mask (1, L)) of the empty prompt: what T5's tokenizer gives for "" padded to `max_length`
    (input ids [eos = 1, pad = 0, ...], mask [1, 0, ...]; ids from `transformers.T5Config`'s defaults) through `t5`, e.g.
    the native `t5.T5EncoderModel`.  Replaces the reference's `null_embed_diffusers_{L}token_fp32.pth` (:444-465)."""
    if max_length < 1:
        raise ValueError("max_length must be >= 1")
    ids = torch.zeros((1, max_length), dtype=torch.long)
    ids[0, 0] = 1
    mask = torch.zeros((1, max_length), dtype=torch.long)
    mask[0, 0] = 1
    dev = getattr(t5, "device", None)
    if dev is not None:
        ids, mask = ids.to(dev), mask.to(dev)
    y = t5(ids, attention_mask=mask)["last_hidden_state"]
    return y[:, None], mask


def _x0_scalars(ac: torch.Tensor, t: int) -> Dict[str, float]:
    """`pxa_lcm_step` as eps_to_mu at t: x0 = (x - sqrt(1 - a) eps) / sqrt(a) with the float32 scalars of the reference."""
    a = ac[t]
    return dict(sqrt_alpha=float(a.sqrt()), sqrt_beta=float((1 - a).sqrt()), c_skip=0.0, c_out=1.0, c_prev=1.0, c_noise=0.0)


def _latents_info(model, x: torch.Tensor, data_info):
    """`forward_model`'s added_cond_kwargs (generate.py:45-52) for a micro-conditioned model: the LATENT h, w and h / w."""
    if data_info is not None or not getattr(model, "micro_conditioning", False):
        return data_info
    b, _, h, w = x.shape
    return dict(img_hw=torch.tensor([[float(h), float(w)]], device=x.device).repeat(b, 1),
                aspect_ratio=torch.tensor([[float(h / w)]], device=x.device).repeat(b, 1))


# ================================================================================================= sampler
class DMDSampler:
    """One-step DMD sampling for a batch of n: `model_fn(x, ts, **model_kwargs)[:, :4]` at int64 ts = `timestep` of shape (n,),
    then x0 = (x - sqrt(1 - a) eps) / sqrt(a) in one `pxa_lcm_step`; returns fp32 latents.  timestep 400 is the app's
    sampler, 999 the training script's `generate_sample_1step`."""

    def __init__(self, model_fn: Callable, timestep: int = 400, num_train_timesteps: int = 1000):
        if not 0 <= int(timestep) < num_train_timesteps:
            raise ValueError(f"timestep must be in [0, {num_train_timesteps})")
        self.model, self.timestep = model_fn, int(timestep)
        self.scalars = _x0_scalars(ddpm_alphas_cumprod(num_train_timesteps), self.timestep)
        self._graphs = CapturedLoops()

    def _run(self, x, den, ts, model_kwargs):
        out = self.model(x, ts, **model_kwargs)
        lib.lcm_step(step_input(out[:, :4]), x, None, den, x, **self.scalars)
        return den

    @torch.no_grad()
    def sample(self, x_T: torch.Tensor, model_kwargs: Optional[dict] = None, cuda_graph: bool = False) -> torch.Tensor:
        """x_T (n, 4, h, w) on the device."""
        model_kwargs = dict(model_kwargs or {})
        if not x_T.is_cuda:
            raise RuntimeError("pixart_sigma_b200.dmd has no CPU path: x_T must be a CUDA tensor")
        if x_T.dim() != 4 or x_T.shape[1] != 4 or (x_T.shape[2] * x_T.shape[3]) % 4:
            raise ValueError("x_T must be (n, 4, h, w) latents with h*w a multiple of 4")
        ts = torch.full((x_T.shape[0],), self.timestep, dtype=torch.int64, device=x_T.device)

        def loop(x0, k, draws):
            x = x0.to(torch.float32).contiguous().clone()
            return self._run(x, torch.empty_like(x), ts, model_kwargs)
        if cuda_graph:                                     # the timestep is fixed per sampler: no extras in the key
            return self._graphs.sample(self.model, model_kwargs, (), x_T, None, loop, (ts,))
        return loop(x_T, None, None)


# ================================================================================================= distillation
class _DmdLoss(torch.autograd.Function):
    """dm_loss over `pxa_dmd_loss`; the gradient with respect to the generator's output is written by the same launches."""

    @staticmethod
    def forward(ctx, gen_out, latents, noisy, t, ac, real_out, fake_out, partials, weight, cfg, sqrt_alpha, sqrt_beta):
        d = torch.empty(gen_out.shape, dtype=torch.float32, device=gen_out.device)
        loss = torch.empty((), dtype=torch.float32, device=gen_out.device)
        lib.dmd_loss(latents, noisy, t, ac, real_out, fake_out, d, loss, weight, partials, cfg=cfg, gen_sqrt_alpha=sqrt_alpha,
                     gen_sqrt_beta=sqrt_beta)
        ctx.save_for_backward(d)
        return loss

    @staticmethod
    def backward(ctx, grad):
        (d,) = ctx.saved_tensors
        return (d * grad,) + (None,) * 11


def _fp32_reducer(reducer, what: str):
    reducer.flatten_params()
    flats = [b["flat_param"] for b in reducer.buckets]
    if not flats or any(not f.is_cuda or f.dtype != torch.float32 for f in flats):
        raise RuntimeError(f"DMDDistiller: the {what}'s reducer must hold fp32 CUDA parameters (use model.float().cuda())")
    return flats[0].device


class DMDDistiller:
    """Distribution-matching distillation (train_pixart_dmd.py:484-697) on the native kernels; see the module docstring.

    generator / fake: the one-step generator and the fake-score model (fp32 master parameters, train mode), whose gradients
    `gen_reducer` / `fake_reducer` (parallel.GradBucketReducer) bucket; their parameters are flattened here.  real: the frozen
    teacher (default: a bf16 copy of the generator, which is where the recipe starts).  uncond_y / uncond_mask: the
    unconditional caption (`null_caption`), (1, [1,] L, C) and (1, L).  cfg: the real model's guidance scale.  one_step_t: the
    generator's timestep; start_ts: timesteps are drawn from [1, start_ts); fix_noise_ts: a fixed timestep instead.
    ema: the EMA model (default: a bf16 copy of the generator), kept as an fp32 master in the generator reducer's layout.
    latent_hw: the latent size of the drawn init_noise (default: the generator's input size)."""

    def __init__(self, generator: torch.nn.Module, gen_reducer, fake: torch.nn.Module, fake_reducer,
                 uncond_y: torch.Tensor, uncond_mask: Optional[torch.Tensor], real: Optional[torch.nn.Module] = None,
                 cfg: float = 3.0, one_step_t: int = 999, start_ts: int = 999, fix_noise_ts: Optional[int] = None,
                 ema: Optional[torch.nn.Module] = None, ema_max_decay: float = 0.9999, use_regression: bool = False,
                 snr_gamma: Optional[float] = None, noise_offset: float = 0.0, num_train_timesteps: int = 1000,
                 latent_hw: Optional[Tuple[int, int]] = None):
        if use_regression:
            raise NotImplementedError("use_regression (the LPIPS regression loss) is not supported")
        if snr_gamma is not None:
            raise NotImplementedError("snr_gamma is not supported")
        if noise_offset != 0:
            raise NotImplementedError("noise_offset is not supported")
        T = int(num_train_timesteps)
        if not 0 <= int(one_step_t) < T:
            raise ValueError(f"one_step_t must be in [0, {T})")
        if not 1 < int(start_ts) <= T:
            raise ValueError(f"start_ts must be in [2, {T}] (timesteps are drawn from [1, start_ts))")
        if fix_noise_ts is not None and not 0 <= int(fix_noise_ts) < T:
            raise ValueError(f"fix_noise_ts must be in [0, {T})")
        if not 0.0 <= ema_max_decay <= 1.0:
            raise ValueError("ema_max_decay must be in [0, 1]")
        for m, what in ((generator, "generator"), (fake, "fake model")):
            if getattr(getattr(m, "y_embedder", None), "uncond_prob", 0.0) > 0:
                raise ValueError(f"DMDDistiller: the {what} was built with class_dropout_prob > 0; the recipe's diffusers "
                                 "transformer drops no captions (build it with class_dropout_prob=0)")
        uy = uncond_y[:, None] if uncond_y.dim() == 3 else uncond_y
        if uy.dim() != 4 or uy.shape[:2] != (1, 1):
            raise ValueError("uncond_y must be one caption: (1, L, C) or (1, 1, L, C)")
        um = None if uncond_mask is None else uncond_mask.reshape(1, -1)
        if um is not None and um.shape[1] != uy.shape[2]:
            raise ValueError(f"uncond_mask must have {uy.shape[2]} entries")
        self.generator, self.gen_reducer, self.fake, self.fake_reducer = generator, gen_reducer, fake, fake_reducer
        self.device = _fp32_reducer(gen_reducer, "generator")
        if _fp32_reducer(fake_reducer, "fake model") != self.device:
            raise RuntimeError("DMDDistiller: the generator and the fake model must be on one device")
        dev = self.device
        self.uncond_y, self.uncond_mask = uy.to(dev), None if um is None else um.to(dev)
        self.cfg, self.one_step_t, self.start_ts = float(cfg), int(one_step_t), int(start_ts)
        self.fix_noise_ts = None if fix_noise_ts is None else int(fix_noise_ts)
        self.ema_max_decay = float(ema_max_decay)
        self.latent_hw = tuple(latent_hw) if latent_hw is not None else (generator.base_size * generator.patch_size,) * 2
        self.alphas_cumprod = ddpm_alphas_cumprod(T)
        self.ac = self.alphas_cumprod.to(dev)                                        # uploaded once
        self.gen_scalars = _x0_scalars(self.alphas_cumprod, self.one_step_t)
        self.real = real if real is not None else _inference_copy(generator)
        self.real.requires_grad_(False)
        self._flat_ema = FlatEMA(generator, gen_reducer, ema, owner="DMDDistiller")
        self.ema_updates = 0
        # the fake model's denoising loss through pxa_lcm_consistency_loss (see _eps_mse): one row, uploaded once
        row = lib.LcmRow(sra_s=0.0, srm1_s=-1.0, cskip_s=0.0, cout_s=1.0, sra_t=0.0, srm1_t=0.0, cskip_t=1.0, cout_t=0.0,
                         sqrt_acp=0.0, sqrt_1macp=0.0)
        self._mse_table = _upload((lib.LcmRow * 1)(row), dev)
        self._mse_partials = torch.empty(lib.LCM_LOSS_PARTS, dtype=torch.float64, device=dev)
        self._ws: Dict[int, tuple] = {}

    ema = property(lambda self: self._flat_ema.ema)

    # ---- EMA: diffusers' EMAModel.step on the generator (train_pixart_dmd.py:696-697)
    @torch.no_grad()
    def update_ema(self) -> None:
        """One `EMAModel.step(generator.parameters())` with the decay of `ema_decay` (host counter): one `pxa_ema_flat` launch
        that writes the fp32 master and the EMA model's bf16 weights.  diffusers' `s -= (1 - d) (s - p)` and the kernel's
        `s d + p (1 - d)` are the same update up to rounding."""
        self.ema_updates += 1
        self._flat_ema.update(ema_decay(self.ema_updates, self.ema_max_decay))

    def ema_state_dict(self) -> Dict[str, torch.Tensor]:
        """The EMA model's state dict with every bucketed parameter as its fp32 master value."""
        return self._flat_ema.state_dict()

    # ---- one step
    def draw(self, b: int, hw: Optional[Sequence[int]] = None):
        """(init_noise, noise, t, noise_f, t_f) from the device generator in the reference's order (`dmd_draws`)."""
        return dmd_draws(b, hw or self.latent_hw, self.device, self.start_ts, self.fix_noise_ts)

    def add_noise(self, x: torch.Tensor, noise: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """`DDPMScheduler.add_noise` (float32 alphas_cumprod): sqrt(a_t) x + sqrt(1 - a_t) noise."""
        return ddpm_add_noise(self.ac, x, noise, t)

    def _workspace(self, b: int):
        if b not in self._ws:
            self._ws[b] = (torch.empty(2 * b * lib.DMD_PARTS, dtype=torch.float64, device=self.device),
                           torch.empty(b, dtype=torch.float32, device=self.device),
                           torch.zeros(b, dtype=torch.int64, device=self.device))
        return self._ws[b]

    def _eps_mse(self, out: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        # mse(out[:, :4], target) and its gradient: the L2 consistency loss over a row that makes model_pred = eps and the
        # target = x_prev exactly (cskip_s 0, cout_s 1, sra_s 0, srm1_s -1; cskip_t 1, cout_t 0); ema_out is multiplied by 0
        index = self._workspace(out.shape[0])[2]
        return _ConsistencyLoss.apply(out, step_input(out.detach()), target, target, index, self._mse_table,
                                      self._mse_partials, lib.LCM_L2, 1.0)

    def step(self, y: torch.Tensor, mask: Optional[torch.Tensor] = None, data_info=None, draws=None,
             loss_scale: float = 1.0) -> Tuple[torch.Tensor, torch.Tensor]:
        """Both forward / backward passes of one step: the generator's gradient of dm_loss into `gen_reducer` and the fake
        model's gradient of its denoising loss into `fake_reducer` (zero both first; calling `step` k times before the
        optimizer steps accumulates).  y (b, 1, L, C) captions, mask (b, L); draws: given `draw()` outputs.  Returns
        (dm_loss, sg_loss) as 0-d device tensors; no host sync.  `self.weight` holds the per-sample DM weight afterwards."""
        from . import autograd as ag
        if y.dim() != 4 or not y.is_cuda:
            raise ValueError("y must be (b, 1, L, C) CUDA caption features")
        b = y.shape[0]
        if y.shape[2] != self.uncond_y.shape[2]:
            raise ValueError(f"captions have {y.shape[2]} tokens, the unconditional caption {self.uncond_y.shape[2]}")
        if (mask is None) != (self.uncond_mask is None):
            raise ValueError("give a caption mask exactly when the unconditional caption has one")
        init_noise, noise, t, noise_f, t_f = draws if draws is not None else self.draw(b)
        if init_noise.shape[0] != b or init_noise.dim() != 4 or init_noise.shape[1] != 4:
            raise ValueError(f"init_noise must be ({b}, 4, h, w)")
        init_noise = init_noise.to(device=self.device, dtype=torch.float32).contiguous()
        t = t.to(device=self.device, dtype=torch.int64).contiguous()
        t_f = t_f.to(device=self.device, dtype=torch.int64)
        di = _latents_info(self.generator, init_noise, data_info)
        partials, weight, _ = self._workspace(b)
        self.gen_reducer.start()
        self.fake_reducer.start()
        # 1. generator: one forward at one_step_t, x0 from its eps (generate_sample_1step)
        ag.refresh_shadows(self.generator)
        t_g = torch.full((b,), self.one_step_t, dtype=torch.int64, device=self.device)
        out_g = self.generator(init_noise, t_g, y, mask=mask, data_info=di)
        if out_g.dtype != torch.float32:
            out_g = out_g.float()
        with torch.no_grad():
            latents, scratch = torch.empty_like(init_noise), torch.empty_like(init_noise)
            lib.lcm_step(step_input(out_g[:, :4]), init_noise, None, latents, scratch, **self.gen_scalars)
            noisy = self.add_noise(latents, noise.to(latents.device), t).contiguous()
            # 2. the real model at batch 2b over [uncond ; cond]
            uy = self.uncond_y.to(dtype=y.dtype).expand(b, *self.uncond_y.shape[1:])
            m2 = None if mask is None else torch.cat([self.uncond_mask.to(mask.dtype).expand(b, -1), mask.reshape(b, -1)])
            di2 = None if di is None else {k: _dup(v) if isinstance(v, torch.Tensor) and v.shape[0] == b else v
                                           for k, v in di.items()}
            real_out = self.real(torch.cat([noisy, noisy]), torch.cat([t, t]), torch.cat([uy, y]), mask=m2, data_info=di2)
        # the fake model's score: on the training path (the fp32 master is not an inference model), detached
        ag.refresh_shadows(self.fake)
        fake_out = self.fake(noisy, t, y, mask=mask, data_info=di).detach()
        dm = _DmdLoss.apply(out_g, latents, noisy, t, self.ac, step_input(real_out), step_input(fake_out), partials, weight,
                            self.cfg, self.gen_scalars["sqrt_alpha"], self.gen_scalars["sqrt_beta"])
        (dm * loss_scale if loss_scale != 1.0 else dm).backward()
        del fake_out, real_out
        # 3. the fake model's denoising loss on the detached x0
        noisy_f = self.add_noise(latents, noise_f.to(latents.device), t_f)
        out_f = self.fake(noisy_f, t_f, y, mask=mask, data_info=di)
        if out_f.dtype != torch.float32:
            out_f = out_f.float()
        sg = self._eps_mse(out_f, noise_f.to(device=self.device, dtype=torch.float32).contiguous())
        (sg * loss_scale if loss_scale != 1.0 else sg).backward()
        self.gen_reducer.finish()
        self.fake_reducer.finish()
        self.latents, self.weight = latents, weight
        return dm.detach(), sg.detach()
