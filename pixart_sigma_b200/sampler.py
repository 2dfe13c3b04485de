"""H100-native driver of the DPM-Solver++ sampling loop around the denoiser hot path (SURVEY.md §8f.1).

Mirrors the reference's `diffusion.DPMS(...)` factory and `DPM_Solver.sample(...)` as `scripts/inference.py:102-118` uses
them (`diffusion/dpm_solver.py:6-35`, `diffusion/model/dpm_solver.py:1069-1241`): same call signature, same result, for
the configuration the reference ships (noise-prediction model, classifier-free guidance, linear discrete schedule,
`algorithm_type="dpmsolver++"`, `method="multistep"`, `order<=2`, `skip_type="time_uniform"`).  Other options raise
`NotImplementedError` instead of silently taking a different path.

What is different from the reference loop:
  * all schedule look-ups (the reference's `interpolate_fn` sorts a 1001-element array on the GPU for every alpha /
    sigma / lambda it needs, ~10 tiny kernels + syncs per step) are done ONCE on the host: per step five scalars;
  * CFG combine, data prediction and the first / second-order multistep update are ONE elementwise sm_90a kernel per
    step (`pxa_dpm_solver_pp_step`, include/pixart_sm100.h) instead of ~25 PyTorch elementwise launches;
  * `cuda_graph=True` captures the whole `steps`-step loop (denoiser launches included) into one CUDA graph.
There is no CPU path: inputs must live on an sm_90 device.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch

from . import lib
from .capture import CapturedLoops, CfgCond, step_input

__all__ = ["DPMS", "DPMSolverPP"]


def linear_betas(diffusion_steps: int = 1000) -> np.ndarray:
    """float64 linear beta schedule (diffusion/model/gaussian_diffusion.py:82,107-116)."""
    scale = 1000 / diffusion_steps
    return np.linspace(scale * 0.0001, scale * 0.02, diffusion_steps, dtype=np.float64)


class _DiscreteVPSchedule:
    """log(alpha) of the discrete linear-beta VP schedule at t_i = i/N (float32 table, piecewise-linear look-up with the
    outermost segments extended), as `NoiseScheduleVP('discrete', betas=linear)` defines it
    (diffusion/model/dpm_solver.py:97-106,127-155; betas: diffusion/model/gaussian_diffusion.py:82,107-116), or of a given
    log(alpha) table at the same times (the SA-Solver's, diffusion/model/sa_solver.py:81-90)."""

    def __init__(self, diffusion_steps: int = 1000, clipped_lambda: float = -5.1, log_alpha: Optional[torch.Tensor] = None):
        if log_alpha is None:
            log_alphas = 0.5 * torch.log(1 - torch.from_numpy(linear_betas(diffusion_steps))).cumsum(dim=0)
            lambs = log_alphas - 0.5 * torch.log(1. - torch.exp(2. * log_alphas))
            drop = int(torch.searchsorted(torch.flip(lambs, [0]), torch.tensor(clipped_lambda, dtype=lambs.dtype)))
            if drop > 0:                       # log-SNR clipped near t = T (a no-op for the linear schedule)
                log_alphas = log_alphas[:-drop]
            log_alpha = log_alphas
        self.log_alpha = log_alpha.to(torch.float32)      # a given table is used as is: no clipping
        self.total_N = self.log_alpha.numel()
        self.t = torch.linspace(0., 1., self.total_N + 1)[1:].to(torch.float32)
        self.T = 1.0

    def log_alpha_at(self, t: torch.Tensor) -> torch.Tensor:
        t = t.reshape(-1).to(torch.float32)
        seg = (torch.searchsorted(self.t, t.contiguous()) - 1).clamp(0, self.total_N - 2)
        t0, t1, y0, y1 = self.t[seg], self.t[seg + 1], self.log_alpha[seg], self.log_alpha[seg + 1]
        return y0 + (t - t0) * (y1 - y0) / (t1 - t0)

    def alpha(self, t):
        return torch.exp(self.log_alpha_at(t))

    def sigma(self, t):
        return torch.sqrt(1. - torch.exp(2. * self.log_alpha_at(t)))

    def lam(self, t):
        la = self.log_alpha_at(t)
        return la - 0.5 * torch.log(1. - torch.exp(2. * la))


class DPMSolverPP:
    """Multistep DPM-Solver++ (order 1 / 2) with classifier-free guidance; see the module docstring."""

    def __init__(self, model: Callable, condition: torch.Tensor, uncondition: Optional[torch.Tensor], cfg_scale: float,
                 model_kwargs: Optional[dict] = None, diffusion_steps: int = 1000):
        self.model = model
        self.condition = condition
        self.uncondition = uncondition
        self.cfg_scale = float(cfg_scale)
        self.model_kwargs = dict(model_kwargs or {})
        self.schedule = _DiscreteVPSchedule(diffusion_steps)
        self._graphs = CapturedLoops()
        self._cfg_cond = CfgCond()

    # ---- host side: everything that does not depend on the latents
    def plan(self, steps: int, order: int = 2, t_start: Optional[float] = None, t_end: Optional[float] = None,
             lower_order_final: bool = True) -> List[dict]:
        """Per update i (time ts[i] -> ts[i+1]): the model-input time and the five scalars of pxa_dpm_solver_pp_step."""
        sch = self.schedule
        t_0 = 1. / sch.total_N if t_end is None else t_end
        t_T = sch.T if t_start is None else t_start
        assert t_0 > 0 and t_T > 0, "time range must be positive (discrete-time DPMs: [1/N, 1])"
        assert steps >= order
        ts = torch.linspace(t_T, t_0, steps + 1)                       # time_uniform (dpm_solver.py:475-476)
        plan = []
        for i in range(steps):
            s, t = ts[i:i + 1], ts[i + 1:i + 2]
            step = i + 1
            step_order = 1 if step < order else (min(order, steps + 1 - step) if lower_order_final else order)
            h = sch.lam(t) - sch.lam(s)
            b = torch.exp(sch.log_alpha_at(t)) * torch.expm1(-h)        # alpha_t * phi_1
            c = torch.zeros_like(b)
            if step_order == 2:
                r0 = (sch.lam(s) - sch.lam(ts[i - 1:i])) / h
                c = 0.5 * b * (1. / r0)
            plan.append(dict(t_input=float((s - 1. / sch.total_N) * 1000.), sigma_s=float(sch.sigma(s)),
                             alpha_s=float(sch.alpha(s)), a=float(sch.sigma(t) / sch.sigma(s)), b=float(b), c=float(c),
                             order=step_order))
        return plan

    # ---- device side
    def _run(self, x: torch.Tensor, x0_prev: torch.Tensor, plan: List[dict], t_dev: List[torch.Tensor], cond: torch.Tensor,
             inter: Optional[list]) -> torch.Tensor:
        n = x.shape[0]
        guided = self.uncondition is not None and self.cfg_scale != 1.
        for st, t_in in zip(plan, t_dev):
            if guided:
                out = self.model(torch.cat([x, x]), t_in, cond, **self.model_kwargs)
            else:                                   # reference: a single conditional evaluation (dpm_solver.py:327-328)
                out = self.model(x, t_in[:n], cond, **self.model_kwargs)
                out = torch.cat([out, out])
            lib.dpm_solver_pp_step(step_input(out), x, x0_prev, cfg_scale=self.cfg_scale if guided else 1.0,
                                   sigma_s=st["sigma_s"], alpha_s=st["alpha_s"], a=st["a"], b=st["b"], c=st["c"])
            if inter is not None:
                inter.append(x.clone())
        return x

    @torch.no_grad()
    def sample(self, x: torch.Tensor, steps: int = 20, t_start: Optional[float] = None, t_end: Optional[float] = None,
               order: int = 2, skip_type: str = "time_uniform", method: str = "multistep", lower_order_final: bool = True,
               denoise_to_zero: bool = False, solver_type: str = "dpmsolver", atol: float = 0.0078, rtol: float = 0.05,
               return_intermediate: bool = False, cuda_graph: bool = False):
        if method != "multistep" or skip_type != "time_uniform" or solver_type != "dpmsolver" or denoise_to_zero or order > 2:
            raise NotImplementedError("only method='multistep', skip_type='time_uniform', solver_type='dpmsolver', "
                                      "order <= 2, denoise_to_zero=False (the configuration scripts/inference.py uses)")
        if not x.is_cuda:
            raise RuntimeError("pixart_sigma_b200.sampler has no CPU path: x must be a CUDA tensor")
        if x.dim() != 4 or x.shape[1] != 4 or (x.shape[2] * x.shape[3]) % 4:
            raise ValueError("x must be (n, 4, h, w) latents with h*w a multiple of 4")
        plan = self.plan(steps, order, t_start, t_end, lower_order_final)
        n = x.shape[0]
        guided = self.uncondition is not None and self.cfg_scale != 1.
        cond = self._cfg_cond(self.uncondition, self.condition) if guided else self.condition    # dpm_solver.py:330
        t_dev = [torch.full((2 * n,), st["t_input"], dtype=torch.float32, device=x.device) for st in plan]
        inter = [] if return_intermediate else None

        def loop(x0, k, draws):
            xs = x0.to(torch.float32).contiguous().clone()
            return self._run(xs, torch.empty_like(xs), plan[:k], t_dev[:k], cond, inter)
        if cuda_graph and not return_intermediate:
            # every per-step scalar, the step orders and t_input are baked into the captured kernel arguments
            extras = (self.cfg_scale, cond.data_ptr(), tuple(cond.shape), tuple(tuple(st.values()) for st in plan))
            out = self._graphs.sample(self.model, self.model_kwargs, extras, x, None, loop, (cond, t_dev))
        else:
            out = loop(x, None, None)
        out = out.to(x.dtype)
        return (out, inter) if return_intermediate else out


def DPMS(model: Callable, condition: torch.Tensor, uncondition: Optional[torch.Tensor], cfg_scale: float,
         model_type: str = "noise", noise_schedule: str = "linear", guidance_type: str = "classifier-free",
         model_kwargs: Optional[dict] = None, diffusion_steps: int = 1000) -> DPMSolverPP:
    """Same signature as the reference factory (`diffusion/dpm_solver.py:6-35`); returns an object with `.sample(...)`."""
    if model_type != "noise" or noise_schedule != "linear" or guidance_type != "classifier-free":
        raise NotImplementedError("only model_type='noise', noise_schedule='linear', guidance_type='classifier-free' "
                                  "(what scripts/inference.py uses)")
    return DPMSolverPP(model, condition, uncondition, cfg_scale, model_kwargs, diffusion_steps)
