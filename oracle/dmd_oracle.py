"""TEST INFRASTRUCTURE ONLY -- plain-torch restatement of the reference's DMD pieces (read from, not copied from, the
reference checkout), pinned against the unmodified reference by oracle/gen_golden_dmd.py -> tests/golden/dmd_*.pt:

  * the float32 DDPMScheduler alphas_cumprod and its add_noise              diffusers (not in the reference tree; restated)
  * eps_to_mu / generate_sample_1step                                        scripts/DMD/transformer_train/generate.py:22-41
  * the distribution-matching loss (use_dm, snr_gamma=None)                  train_scripts/train_pixart_dmd.py:493-571
  * the fake model's denoising loss                                          train_scripts/train_pixart_dmd.py:627-669
  * EMAModel.step with its decay (0, then min((1 + s) / (10 + s), 0.9999))   diffusers training_utils (restated, unpinned)
Only tests and the fixture generator import this module; the product (`pixart_sigma_b200/dmd.py`) must not.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch
import torch.nn.functional as F

from oracle.lcm_oracle import alphas_cumprod  # noqa: F401  (the same float32 linear-beta table)


def add_noise(ac: torch.Tensor, x: torch.Tensor, noise: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    a = ac.to(x.dtype)[t]
    return (a ** 0.5).flatten().view(-1, 1, 1, 1) * x + ((1 - a) ** 0.5).flatten().view(-1, 1, 1, 1) * noise


def eps_to_mu(ac: torch.Tensor, eps: torch.Tensor, x: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
    a = ac.to(x.dtype)[t].view(-1, 1, 1, 1)
    return (x - (1 - a) ** 0.5 * eps) / a ** 0.5


def sample(model: Callable, x: torch.Tensor, t: int, ac: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One-step sampling: model(x, ts)[:, :4] at ts = t, then eps_to_mu."""
    ac = alphas_cumprod() if ac is None else ac
    ts = torch.full((x.shape[0],), t, dtype=torch.long)
    return eps_to_mu(ac, model(x, ts)[:, :4].float(), x, torch.tensor([t]))


def dm_loss(latents, noisy, t, real_out, fake_out, ac, cfg: float = 3.0) -> Dict[str, torch.Tensor]:
    """real_out: (2b, >=4, h, w) over [uncond ; cond]; fake_out: (b, >=4, h, w).  dm_loss keeps latents' graph."""
    b = latents.shape[0]
    su, sc = (-real_out[:, :4].float()).chunk(2)
    score_real = su + cfg * (sc - su)
    score_fake = -fake_out[:, :4].float()
    a = ac.to(latents.dtype)[t]
    beta = 1.0 - a
    coeff = (score_fake - score_real) * beta.view(-1, 1, 1, 1) ** 0.5 / a.view(-1, 1, 1, 1) ** 0.5
    pred = (noisy + beta.view(-1, 1, 1, 1) ** 0.5 * score_real) / a.view(-1, 1, 1, 1) ** 0.5
    weight = 1. / ((latents - pred).abs().mean([1, 2, 3], keepdim=True) + 1e-5).detach()
    loss = F.mse_loss(latents, (latents - weight * coeff).detach())
    return dict(coeff=coeff, pred=pred, weight=weight.reshape(b), dm_loss=loss)


def step(generator: Callable, real: Callable, fake: Callable, y, mask, uncond_y, uncond_mask, draws, cfg: float = 3.0,
         one_step_t: int = 999, ac: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """One DMD step's tensors.  model(x, t, y, mask) -> (b, 8, h, w); generator and fake keep their graphs (dm_loss and
    sg_loss can be differentiated); uncond_y (1, 1, L, C), uncond_mask (1, L)."""
    ac = alphas_cumprod() if ac is None else ac
    init_noise, noise, t, noise_f, t_f = draws
    b = init_noise.shape[0]
    eps_g = generator(init_noise, torch.full((b,), one_step_t, dtype=torch.long), y, mask)[:, :4]
    latents = eps_to_mu(ac, eps_g, init_noise, torch.tensor([one_step_t]))
    noisy = add_noise(ac, latents, noise, t)
    with torch.no_grad():
        m2 = None if mask is None else torch.cat([uncond_mask.expand(b, -1).to(mask.dtype), mask])
        real_out = real(torch.cat([noisy, noisy]), torch.cat([t, t]), torch.cat([uncond_y.expand(b, -1, -1, -1), y]), m2)
        fake_out = fake(noisy, t, y, mask)
    r = dm_loss(latents, noisy, t, real_out, fake_out, ac, cfg)
    noisy_f = add_noise(ac, latents.detach(), noise_f, t_f)
    sg = F.mse_loss(fake(noisy_f, t_f, y, mask)[:, :4].float(), noise_f.float())
    return dict(latents=latents, noisy=noisy, real_out=real_out, fake_out=fake_out, sg_loss=sg, **r)


def ema_decay(update: int, max_decay: float = 0.9999) -> float:
    s = max(0, update - 1)
    return 0.0 if s <= 0 else min((1 + s) / (10 + s), max_decay)


@torch.no_grad()
def ema_step(shadow: Dict[str, torch.Tensor], params: Dict[str, torch.Tensor], decay: float) -> None:
    one_minus_decay = 1 - decay
    for k, s in shadow.items():
        s.sub_(one_minus_decay * (s - params[k]))
