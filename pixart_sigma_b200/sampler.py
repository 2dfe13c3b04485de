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

from typing import Callable, Dict, List, Optional

import numpy as np
import torch

from . import lib

__all__ = ["DPMS", "DPMSolverPP"]


def linear_betas(diffusion_steps: int = 1000) -> np.ndarray:
    """float64 linear beta schedule (diffusion/model/gaussian_diffusion.py:82,107-116)."""
    scale = 1000 / diffusion_steps
    return np.linspace(scale * 0.0001, scale * 0.02, diffusion_steps, dtype=np.float64)


def _denoiser_params(model: Callable) -> list:
    owner = getattr(model, "__self__", model)              # the nn.Module behind a bound forward_with_dpmsolver
    return list(owner.parameters()) if isinstance(owner, torch.nn.Module) else []


def _denoiser_key(model: Callable, params: list, model_kwargs: Optional[dict]) -> tuple:
    """The denoiser's part of a captured sampling loop's cache key.  `model_kwargs` tensors are captured by address, and so
    are the denoiser's parameters: the fused-LN forward keeps tables derived from them that a replay cannot refresh."""
    kw_id = tuple(sorted((k, (v.data_ptr(), tuple(v.shape)) if isinstance(v, torch.Tensor) else repr(v))
                         for k, v in (model_kwargs or {}).items()))
    owner = getattr(model, "__self__", model)
    derived = getattr(owner, "_ln_fusion", None) is not None
    wkey = (sum(p._version for p in params), params[0].data_ptr()) if (params and derived) else None
    return kw_id, wkey


def _capture(warmup: Callable[[], None], body: Callable[[], None]) -> torch.cuda.CUDAGraph:
    """Run `warmup` eagerly on a side stream (lazy inits, tensor maps), then capture `body` into a CUDA graph."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        warmup()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    return graph


def _step_input(out: torch.Tensor) -> torch.Tensor:
    """The denoiser output as a step kernel reads it: fp32 or bf16 with dense (h, w) planes (channel slices are fine)."""
    if out.dtype not in (torch.float32, torch.bfloat16):
        out = out.float()
    if not (out.stride(3) == 1 and out.stride(2) == out.shape[3] and out.stride(1) == out.shape[2] * out.shape[3]):
        out = out.contiguous()
    return out


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
        self._graphs: Dict[tuple, tuple] = {}
        self._cfg_cond: Optional[torch.Tensor] = None          # cat([uncondition, condition]), built once
        self._params = _denoiser_params(model)

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
            lib.dpm_solver_pp_step(_step_input(out), x, x0_prev, cfg_scale=self.cfg_scale if guided else 1.0,
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
        if guided and self._cfg_cond is None:
            self._cfg_cond = torch.cat([self.uncondition, self.condition])    # [uncond ; cond] (dpm_solver.py:330)
        cond = self._cfg_cond if guided else self.condition
        t_dev = [torch.full((2 * n,), st["t_input"], dtype=torch.float32, device=x.device) for st in plan]
        if cuda_graph and not return_intermediate:
            return self._sample_graphed(x, plan, t_dev, cond)
        xs = x.to(torch.float32).contiguous().clone()
        x0_prev = torch.empty_like(xs)
        inter = [] if return_intermediate else None
        out = self._run(xs, x0_prev, plan, t_dev, cond, inter)
        out = out.to(x.dtype)
        return (out, inter) if return_intermediate else out

    def _sample_graphed(self, x, plan, t_dev, cond):
        # every per-step scalar (sigma_s, alpha_s, a, b, c), the step orders and t_input are baked into the captured kernel
        # arguments, and `cond` / model_kwargs tensors into the captured forward: all of them are part of the key
        kw_id, wkey = _denoiser_key(self.model, self._params, self.model_kwargs)
        key = (tuple(x.shape), x.device.index, float(self.cfg_scale), cond.data_ptr(), tuple(cond.shape), kw_id, wkey,
               tuple((st["t_input"], st["sigma_s"], st["alpha_s"], st["a"], st["b"], st["c"], st.get("order")) for st in plan))
        if key not in self._graphs:
            x_static = x.to(torch.float32).contiguous().clone()
            x0_prev = torch.empty_like(x_static)
            z_in = torch.empty_like(x_static)

            def body():
                x_static.copy_(z_in)
                self._run(x_static, x0_prev, plan, t_dev, cond, None)
            graph = _capture(lambda: self._run(x_static, x0_prev, plan[:2], t_dev[:2], cond, None), body)
            self._graphs[key] = (graph, z_in, x_static, t_dev, cond)
        graph, z_in, x_static = self._graphs[key][:3]
        z_in.copy_(x)
        graph.replay()
        return x_static.to(x.dtype).clone()


def DPMS(model: Callable, condition: torch.Tensor, uncondition: Optional[torch.Tensor], cfg_scale: float,
         model_type: str = "noise", noise_schedule: str = "linear", guidance_type: str = "classifier-free",
         model_kwargs: Optional[dict] = None, diffusion_steps: int = 1000) -> DPMSolverPP:
    """Same signature as the reference factory (`diffusion/dpm_solver.py:6-35`); returns an object with `.sample(...)`."""
    if model_type != "noise" or noise_schedule != "linear" or guidance_type != "classifier-free":
        raise NotImplementedError("only model_type='noise', noise_schedule='linear', guidance_type='classifier-free' "
                                  "(what scripts/inference.py uses)")
    return DPMSolverPP(model, condition, uncondition, cfg_scale, model_kwargs, diffusion_steps)
