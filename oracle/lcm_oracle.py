"""TEST INFRASTRUCTURE ONLY -- plain-torch restatement of the reference's LCM pieces (read from, not copied from, the
reference checkout), pinned against the unmodified reference by oracle/gen_golden_lcm.py -> tests/golden/lcm_*.pt:

  * LCMScheduler: float32 linear betas / alphas_cumprod, set_timesteps, the epsilon-prediction step with the boundary
    scalings, noise from the CPU default generator at every step when there is more than one timestep
                                                      diffusion/lcm_scheduler.py:176-227, 288-410
  * the sampling loop of log_validation for a batch  train_scripts/train_pixart_lcm.py:105-135
  * DDIMSolver, scalings_for_boundary_conditions, the distillation step with IDDPM(return_startx=True) and ema_update
                                                      train_scripts/train_pixart_lcm.py:48-101, 223-309;
                                                      diffusion/model/gaussian_diffusion.py:744-790
Only tests and the fixture generator import this module; the product (`pixart_sigma_b200/lcm.py`) must not.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional

import numpy as np
import torch


# ------------------------------------------------------------------------------------------------- sampler
def scalings(t: torch.Tensor):
    """c_skip, c_out with sigma_data 0.5 and t / 0.1 (float32 on an int64 tensor)."""
    c_skip = 0.25 / ((t / 0.1) ** 2 + 0.25)
    c_out = (t / 0.1) / ((t / 0.1) ** 2 + 0.25) ** 0.5
    return c_skip, c_out


def alphas_cumprod(num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02) -> torch.Tensor:
    betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    return torch.cumprod(1.0 - betas, dim=0)


def lcm_timesteps(steps: int, origin_steps: int = 50, num_train_timesteps: int = 1000) -> torch.Tensor:
    c = num_train_timesteps // origin_steps
    origin = np.arange(1, origin_steps + 1) * c - 1
    return torch.from_numpy(origin[::-(len(origin) // steps)][:steps].copy())


def lcm_step(model_output, i: int, timesteps: torch.Tensor, sample, ac: torch.Tensor, noise: Optional[torch.Tensor]):
    """One epsilon-prediction step; `noise` is the draw of this step (None with a single timestep)."""
    t = timesteps[i]
    prev_t = timesteps[i + 1] if i + 1 < len(timesteps) else t
    a_t, a_prev = ac[t], ac[prev_t]
    c_skip, c_out = scalings(t)
    x0 = (sample - (1 - a_t).sqrt() * model_output) / a_t.sqrt()
    denoised = c_out * x0 + c_skip * sample
    prev = denoised if noise is None else a_prev.sqrt() * denoised + (1 - a_prev).sqrt() * noise
    return prev, denoised


def sample(model: Callable, x_T: torch.Tensor, steps: int = 4, origin_steps: int = 50, model_kwargs: Optional[dict] = None,
           noise: Optional[torch.Tensor] = None):
    """The log_validation loop for a batch of n: model(x, ts, **kw)[:, :4] then the step.  noise None: drawn from the CPU
    default generator as the reference draws it.  Returns (denoised, draws)."""
    ac = alphas_cumprod()
    ts = lcm_timesteps(steps, origin_steps)
    x = x_T
    draws: List[torch.Tensor] = []
    denoised = None
    for i, t in enumerate(ts):
        out = model(x, torch.full((x.shape[0],), int(t), dtype=torch.long), **(model_kwargs or {}))[:, :4]
        z = None
        if len(ts) > 1:
            z = torch.randn(out.shape) if noise is None else noise[i]
            draws.append(z)
        x, denoised = lcm_step(out.float(), i, ts, x, ac, z)
    return denoised, (torch.stack(draws) if draws else torch.zeros(0))


# ------------------------------------------------------------------------------------------------- distillation
class Schedule:
    """The fp64 IDDPM tables the distillation step reads (linear betas, 1000 steps) and the DDIM solver's."""

    def __init__(self, num_train_timesteps: int = 1000, num_ddim_timesteps: int = 50):
        betas = np.linspace(0.0001, 0.02, num_train_timesteps, dtype=np.float64)
        self.ac = np.cumprod(1.0 - betas)
        self.sqrt_ac, self.sqrt_1mac = np.sqrt(self.ac), np.sqrt(1.0 - self.ac)
        self.sqrt_recip_ac, self.sqrt_recipm1_ac = np.sqrt(1.0 / self.ac), np.sqrt(1.0 / self.ac - 1)
        self.topk = num_train_timesteps // num_ddim_timesteps
        self.ddim_timesteps = torch.from_numpy((np.arange(1, num_ddim_timesteps + 1) * self.topk).round().astype(np.int64) - 1)
        self.acp_prev = torch.from_numpy(np.asarray([self.ac[0]] + self.ac[self.ddim_timesteps[:-1].numpy()].tolist()))

    @staticmethod
    def x(arr: np.ndarray, t: torch.Tensor) -> torch.Tensor:
        return torch.from_numpy(arr)[t].float()[:, None, None, None]


def distill_step(student: Callable, teacher: Callable, ema: Callable, latents, y, mask, noise, index, uncond, w: float = 4.5,
                 huber_c: float = 1e-3, sch: Optional[Schedule] = None) -> Dict[str, torch.Tensor]:
    """One distillation step's tensors (the student's graph is kept: `loss_huber` / `loss_l2` can be differentiated).
    model(x, t, y, mask) returns the 8-channel output."""
    sch = sch or Schedule()
    b = latents.shape[0]
    start = sch.ddim_timesteps[index]
    t = torch.where(start - sch.topk < 0, torch.zeros_like(start), start - sch.topk)
    cs_s, co_s = [v.reshape(b, 1, 1, 1) for v in scalings(start)]
    cs_t, co_t = [v.reshape(b, 1, 1, 1) for v in scalings(t)]
    wt = (w * torch.ones((b,))).reshape(b, 1, 1, 1)
    x_t = sch.x(sch.sqrt_ac, start) * latents + sch.x(sch.sqrt_1mac, start) * noise
    x0 = lambda xx, tt, eps: sch.x(sch.sqrt_recip_ac, tt) * xx - sch.x(sch.sqrt_recipm1_ac, tt) * eps
    eps_s = student(x_t, start, y, mask)[:, :4]
    model_pred = cs_s * x_t + co_s * x0(x_t, start, eps_s)
    with torch.no_grad():
        eps_c, eps_u = teacher(x_t, start, y, mask)[:, :4], teacher(x_t, start, uncond, mask)[:, :4]
        x0_c, x0_u = x0(x_t, start, eps_c), x0(x_t, start, eps_u)
        px0 = x0_c + wt * (x0_c - x0_u)
        peps = eps_c + wt * (eps_c - eps_u)
        acp = sch.acp_prev[index].reshape(b, 1, 1, 1)                            # fp64
        x_prev = acp.sqrt() * px0 + (1.0 - acp).sqrt() * peps                      # fp64
        xp32 = x_prev.float()
        eps_e = ema(xp32, t, y, mask)[:, :4]
        target = cs_t * x_prev + co_t * x0(xp32, t, eps_e)                         # fp64
    d = model_pred.float() - target.float()
    return dict(start=start, t=t, x_t=x_t, eps_s=eps_s, model_pred=model_pred, x_prev=x_prev, eps_e=eps_e, target=target,
                loss_huber=torch.mean(torch.sqrt(d ** 2 + huber_c ** 2) - huber_c),
                loss_l2=torch.nn.functional.mse_loss(model_pred.float(), target.float(), reduction="mean"))


@torch.no_grad()
def ema_update(dest: Dict[str, torch.Tensor], src: Dict[str, torch.Tensor], rate: float) -> None:
    for k, d in dest.items():
        d.mul_(rate).add_((1 - rate) * src[k])
