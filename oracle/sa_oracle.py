"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's SA-Solver sampling loop as `scripts/inference.py` drives it
(`SASolverSampler(model.forward_with_dpmsolver, device=device).sample(S=25, batch_size=n, shape=(4, h, w), eta=1,
conditioning=..., unconditional_conditioning=..., unconditional_guidance_scale=..., model_kwargs=...)`,
scripts/inference.py:119-133).  Only tests may import this module; the product (`pixart_sigma_b200/sa_sampler.py`) must not.

Pinned against the unmodified reference (`diffusion/sa_sampler.py::SASolverSampler`, imported through oracle/refshim.py) by
`oracle/gen_golden_sa.py` -> `tests/golden/sa_*.pt`, checked in tests/test_sa_solver_cpu.py.

What is restated (file:line in the reference, PixArt-alpha/PixArt-sigma), for the one configuration SASolverSampler.sample uses
(mode 'few_steps', skip_type 'time', skip_order 1, predictor_order 2, corrector_order 2, pc_mode 'PEC', data prediction):
  * alphas_cumprod: float64 cumprod of the linear betas, cast to float32     diffusion/sa_sampler.py:19-22
  * NoiseScheduleVP('discrete', alphas_cumprod): log_alpha = 0.5 log(.) in float32, t_i = i / N, no log-SNR clipping,
    piecewise-linear look-ups                                                 diffusion/model/sa_solver.py:81-90,108-140,1099-1137
  * model_wrapper: t_input = (t - 1/N) * 1000, CFG batch [uncond, cond], eps = eu + s (ec - eu); one conditional
    evaluation when s == 1 or there is no unconditional input                 diffusion/model/sa_solver.py:259-318
  * data prediction m = (x - sigma eps) / alpha                               diffusion/model/sa_solver.py:377-386
  * time steps linspace(1, 1/N, S + 1) (skip_order 1)                         diffusion/model/sa_solver.py:408-410
  * exponential-integral and Lagrange coefficients (orders 0-1)               diffusion/model/sa_solver.py:449-505,541-560
  * predictor / corrector with the order-2 "few steps" modification           diffusion/model/sa_solver.py:644-753
  * PEC driver: order-1 predictor at the first and the last step, tau = 0 and no evaluation at the last step, one
    randn_like draw at init and one per step                                  diffusion/model/sa_solver.py:755-897
  * tau(t) = eta on 0.2 <= t <= 0.8, else 0                                   diffusion/sa_sampler.py:90
Every scalar is computed with the reference's float32 torch operations in the reference's order.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch

from oracle import dpm_oracle as do


class SASchedule(do.DiscreteSchedule):
    """`NoiseScheduleVP('discrete', alphas_cumprod=...)` as SASolverSampler builds it (no log-SNR clipping)."""

    def __init__(self, betas: Optional[np.ndarray] = None):
        betas = do.linear_betas() if betas is None else betas
        alphas_cumprod = torch.cumprod(1.0 - torch.tensor(betas), dim=0).to(torch.float32)      # sa_sampler.py:19-22
        self.log_alpha = 0.5 * torch.log(alphas_cumprod)                                        # sa_solver.py:86
        self.total_N = self.log_alpha.numel()
        self.t = torch.linspace(0., 1., self.total_N + 1)[1:].to(torch.float32)
        self.T = 1.0


def time_steps(sch: SASchedule, steps: int) -> torch.Tensor:
    return torch.linspace(sch.T, 1. / sch.total_N, steps + 1).pow(1)


def tau_of(t: torch.Tensor, eta: float):
    return eta if 0.2 <= t <= 0.8 else 0


def _exp_positive(order, start, end, tau):
    """sa_solver.py:449-471, orders 0 and 1."""
    end_cov = (1 + tau ** 2) * end
    start_cov = (1 + tau ** 2) * start
    if order == 0:
        return torch.exp(end_cov) * (1 - torch.exp(-(end_cov - start_cov))) / ((1 + tau ** 2))
    return torch.exp(end_cov) * ((end_cov - 1) - (start_cov - 1) * torch.exp(-(end_cov - start_cov))) / ((1 + tau ** 2) ** 2)


def _gradient_coefficients(order, start, end, lams, tau):
    """sa_solver.py:478-505,541-560 (data prediction)."""
    if order == 1:
        lag = [[1]]
    else:
        lag = [[1 / (lams[0] - lams[1]), -lams[1] / (lams[0] - lams[1])],
               [1 / (lams[1] - lams[0]), -lams[0] / (lams[1] - lams[0])]]
    out = []
    for i in range(order):
        c = 0
        for j in range(order):
            c += lag[i][j] * _exp_positive(order - 1 - j, start, end, tau)
        out.append(c)
    return out


def update_coefficients(sch: SASchedule, ts: torch.Tensor, i: int, order: int, tau, corrector: bool):
    """Scalars of the update to t_i (sa_solver.py:644-753): x_new = A x + K[0] m_a + K[1] m_b + N xi, with
    (m_a, m_b) = (m_{i-1}, m_{i-2}) for the predictor and (m_i, m_{i-1}) for the corrector."""
    t, t_prev = ts[i:i + 1], ts[i - 1:i]
    sigma_t, lambda_t = sch.sigma(t), sch.lam(t)
    sigma_prev, lambda_prev = sch.sigma(t_prev), sch.lam(t_prev)
    h = lambda_t - lambda_prev
    if corrector:
        lams = [lambda_t, lambda_prev][:order]
    else:
        lams = [lambda_prev, sch.lam(ts[i - 2:i - 1]) if order == 2 else None][:order]
    g = _gradient_coefficients(order, lambda_prev, lambda_t, lams, tau)
    if order == 2:
        if corrector:
            mod = 1.0 * torch.exp((1 + tau ** 2) * lambda_t) * (
                h / 2 - (h * (1 + tau ** 2) - 1 + torch.exp((1 + tau ** 2) * (-h))) / ((1 + tau ** 2) ** 2 * h))
        else:
            mod = 1.0 * torch.exp((1 + tau ** 2) * lambda_t) * (
                h ** 2 / 2 - (h * (1 + tau ** 2) - 1 + torch.exp((1 + tau ** 2) * (-h))) / ((1 + tau ** 2) ** 2)) / (
                lambda_prev - sch.lam(ts[i - 2:i - 1]))
        g[0] += mod
        g[1] -= mod
    K = [(1 + tau ** 2) * sigma_t * torch.exp(- tau ** 2 * lambda_t) * g[k] for k in range(order)]
    if order == 1:
        K.append(torch.zeros_like(K[0]))
    N = sigma_t * torch.sqrt(1 - torch.exp(-2 * tau ** 2 * h))
    A = torch.exp(-tau ** 2 * h) * (sigma_t / sigma_prev)
    return A, K, N


def step_coefficients(steps: int, eta: float, sch: Optional[SASchedule] = None) -> List[dict]:
    """Per denoiser evaluation i (0 <= i < steps), the scalars of pxa_sa_solver_step as floats: the data prediction at t_i
    (sigma, alpha), the corrector to x_i (c_*; identity at i = 0) and the predictor to x~_{i+1} (p_*)."""
    assert steps >= 2
    sch = sch or SASchedule()
    ts = time_steps(sch, steps)
    out = []
    for i in range(steps):
        t = ts[i:i + 1]
        d = dict(t_input=float(do.model_input_time(sch, t)), sigma=float(sch.sigma(t)), alpha=float(sch.alpha(t)))
        if i == 0:
            d.update(c_x=1.0, c_m0=0.0, c_m1=0.0, c_noise=0.0)
        else:
            A, K, N = update_coefficients(sch, ts, i, 2, tau_of(ts[i], eta), corrector=True)
            d.update(c_x=float(A), c_m0=float(K[0]), c_m1=float(K[1]), c_noise=float(N))
        j = i + 1
        last = j == steps
        A, K, N = update_coefficients(sch, ts, j, 1 if (j == 1 or last) else 2, 0 if last else tau_of(ts[j], eta),
                                      corrector=False)
        d.update(p_x=float(A), p_m0=float(K[0]), p_m1=float(K[1]), p_noise=float(N))
        out.append(d)
    return out


def sample(model: Callable, x_T: torch.Tensor, condition: torch.Tensor, uncondition: Optional[torch.Tensor],
           cfg_scale: float, steps: int, eta: float, noise: List[torch.Tensor], model_kwargs: Optional[dict] = None,
           return_first_corrected: bool = False):
    """`model(x, t_input, cond, **model_kwargs) -> eps`; `noise`: the draws xi_1 .. xi_steps (the reference's randn_like
    draws after the discarded one at init).  Returns x at t = 1/N (and the corrected x_1)."""
    assert len(noise) == steps
    model_kwargs = model_kwargs or {}
    sch = SASchedule()
    ts = time_steps(sch, steps)
    guided = not (cfg_scale == 1. or uncondition is None)

    def data_pred(x, t):
        t_in = do.model_input_time(sch, t.expand(x.shape[0]))
        if guided:
            out = model(torch.cat([x] * 2), torch.cat([t_in] * 2), torch.cat([uncondition, condition]), **model_kwargs)
            eu, ec = out.to(torch.float32).chunk(2)
            eps = eu + cfg_scale * (ec - eu)
        else:
            eps = model(x, t_in, condition, **model_kwargs).to(torch.float32)
        return (x - sch.sigma(t) * eps) / sch.alpha(t)

    def update(x, A, K, N, ma, mb, xi):
        grad = torch.zeros_like(x)
        grad += K[0] * ma
        if mb is not None:
            grad += K[1] * mb
        return A * x + grad + N * xi

    x = x_T.to(torch.float32)
    ms = [data_pred(x, ts[0:1])]
    first = None
    for i in range(1, steps + 1):
        last = i == steps
        order_p = 1 if (i == 1 or last) else 2
        tau = 0 if last else tau_of(ts[i], eta)
        A, K, N = update_coefficients(sch, ts, i, order_p, tau, corrector=False)
        x_p = update(x, A, K, N, ms[-1], ms[-2] if order_p == 2 else None, noise[i - 1])
        if last:
            x = x_p
            break
        ms.append(data_pred(x_p, ts[i:i + 1]))
        tau = tau_of(ts[i], eta)
        A, K, N = update_coefficients(sch, ts, i, 2, tau, corrector=True)
        x = update(x, A, K, N, ms[-1], ms[-2], noise[i - 1])
        if first is None:
            first = x
        ms = ms[-2:]
    return (x, first) if return_first_corrected else x
