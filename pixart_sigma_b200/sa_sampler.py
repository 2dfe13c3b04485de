"""H100-native driver of the SA-Solver sampling loop around the denoiser hot path.

Mirrors the reference's `diffusion.SASolverSampler` as `scripts/inference.py:119-133` uses it (`diffusion/sa_sampler.py:10-94`,
`diffusion/model/sa_solver.py:755-897`): same constructor, same `.sample(...)` signature, same result and the same use of the
random number generator, for the one configuration the reference ships (`mode='few_steps'`, `skip_type='time'`,
`predictor_order=2`, `corrector_order=2`, `pc_mode='PEC'`, data prediction, `tau(t) = eta` on 0.2 <= t <= 0.8, classifier-free
guidance, linear discrete schedule, noise-prediction model).  Arguments that would change the algorithm raise
`NotImplementedError`.

What is different from the reference loop:
  * every schedule look-up and every Lagrange / exponential-integral coefficient (dozens of 1-element float32 device ops per
    step in the reference, each look-up sorting a 1001-entry table) is computed ONCE on the host, with the reference's float32
    operations in the reference's order: eleven scalars per denoiser evaluation;
  * CFG combine, data prediction, the corrector giving x_i and the predictor giving the next denoiser input are ONE elementwise
    sm_90a kernel per evaluation (`pxa_sa_solver_step`, include/pixart_sm100.h);
  * the stochastic window is decided on the host, so the loop has no host sync and `cuda_graph=True` captures all S
    evaluations, noise draws included, into one CUDA graph (each replay draws fresh noise from the default CUDA generator).
There is no CPU path: inputs must live on an sm_90 device.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence

import torch

from . import lib
from .capture import CapturedLoops, CfgCond, step_input
from .sampler import _DiscreteVPSchedule, linear_betas

__all__ = ["SASolverSampler"]

_STEP_KEYS = ("sigma", "alpha", "c_x", "c_m0", "c_m1", "c_noise", "p_x", "p_m0", "p_m1", "p_noise")


def _tau(t: torch.Tensor, eta: float):
    """diffusion/sa_sampler.py:90, decided on the float32 time step (a host value here, a device sync in the reference)."""
    return eta if 0.2 <= t <= 0.8 else 0


def _exp_positive(order: int, start, end, tau):
    """Integral of exp((1 + tau^2) x) x^order over [start, end], orders 0 and 1 (diffusion/model/sa_solver.py:449-467)."""
    end_cov = (1 + tau ** 2) * end
    start_cov = (1 + tau ** 2) * start
    if order == 0:
        return torch.exp(end_cov) * (1 - torch.exp(-(end_cov - start_cov))) / ((1 + tau ** 2))
    return torch.exp(end_cov) * ((end_cov - 1) - (start_cov - 1) * torch.exp(-(end_cov - start_cov))) / ((1 + tau ** 2) ** 2)


class SASolverSampler:
    """SA-Solver (PEC, predictor and corrector order 2) with classifier-free guidance; see the module docstring."""

    def __init__(self, model: Callable, noise_schedule: str = "linear", diffusion_steps: int = 1000, device="cuda"):
        if noise_schedule != "linear":
            raise NotImplementedError("only noise_schedule='linear' (what scripts/inference.py uses)")
        self.model = model
        self.device = device
        # float64 cumprod cast to float32, then 0.5 * log in float32 (diffusion/sa_sampler.py:19-22, sa_solver.py:86)
        alphas_cumprod = torch.cumprod(1.0 - torch.from_numpy(linear_betas(diffusion_steps)), dim=0).to(torch.float32)
        self.schedule = _DiscreteVPSchedule(log_alpha=0.5 * torch.log(alphas_cumprod))
        self._plans: Dict[tuple, List[dict]] = {}
        self._graphs = CapturedLoops()
        self._cfg_cond = CfgCond()

    # ---- host side: everything that does not depend on the latents
    def _update(self, ts: torch.Tensor, i: int, order: int, tau, corrector: bool):
        """Scalars of the update to t_i (sa_solver.py:644-753): x_new = A x + K[0] m_a + K[1] m_b + N xi with
        (m_a, m_b) = (m_{i-1}, m_{i-2}) for the predictor and (m_i, m_{i-1}) for the corrector."""
        sch = self.schedule
        t, t_prev = ts[i:i + 1], ts[i - 1:i]
        sigma_t, lambda_t = sch.sigma(t), sch.lam(t)
        sigma_prev, lambda_prev = sch.sigma(t_prev), sch.lam(t_prev)
        h = lambda_t - lambda_prev
        lam_other = lambda_t if corrector else (sch.lam(ts[i - 2:i - 1]) if order == 2 else None)
        if order == 1:                                     # Lagrange basis of order 0 (sa_solver.py:485-486)
            g = [0 + 1 * _exp_positive(0, lambda_prev, lambda_t, tau)]
        else:                                              # order 1 (:487-489) on (lambda_t, lambda_prev) / (lambda_prev, lambda_{i-2})
            l0, l1 = (lambda_t, lambda_prev) if corrector else (lambda_prev, lam_other)
            lag = [[1 / (l0 - l1), -l1 / (l0 - l1)], [1 / (l1 - l0), -l0 / (l1 - l0)]]
            e1, e0 = _exp_positive(1, lambda_prev, lambda_t, tau), _exp_positive(0, lambda_prev, lambda_t, tau)
            g = [0 + lag[k][0] * e1 + lag[k][1] * e0 for k in range(2)]
            # the order-2 "few steps" modification (:672-679 predictor, :729-734 corrector), restated op for op in float32
            if corrector:
                mod = 1.0 * torch.exp((1 + tau ** 2) * lambda_t) * (
                    h / 2 - (h * (1 + tau ** 2) - 1 + torch.exp((1 + tau ** 2) * (-h))) / ((1 + tau ** 2) ** 2 * h))
            else:
                mod = 1.0 * torch.exp((1 + tau ** 2) * lambda_t) * (
                    h ** 2 / 2 - (h * (1 + tau ** 2) - 1 + torch.exp((1 + tau ** 2) * (-h))) / ((1 + tau ** 2) ** 2)) / (
                    lambda_prev - lam_other)
            g = [g[0] + mod, g[1] - mod]
        K = [float((1 + tau ** 2) * sigma_t * torch.exp(- tau ** 2 * lambda_t) * gk) for gk in g] + [0.0]
        N = float(sigma_t * torch.sqrt(1 - torch.exp(-2 * tau ** 2 * h)))
        A = float(torch.exp(-tau ** 2 * h) * (sigma_t / sigma_prev))
        return A, K[0], K[1], N

    def plan(self, S: int, eta: float) -> List[dict]:
        """Per denoiser evaluation i (0 <= i < S) at t_i: the model-input time and the scalars of pxa_sa_solver_step -- the
        data prediction (sigma, alpha), the corrector giving x_i (c_*; the identity at i = 0) and the predictor giving
        x~_{i+1} (p_*; order 1 at the first and the last step, tau = 0 at the last: sa_solver.py:804-860)."""
        key = (int(S), float(eta))
        if key in self._plans:
            return self._plans[key]
        if S < 2:
            raise ValueError("SA-Solver with predictor order 2 needs S >= 2 (diffusion/model/sa_solver.py:778)")
        sch = self.schedule
        ts = torch.linspace(sch.T, 1. / sch.total_N, S + 1).pow(1)           # skip_type 'time' (sa_solver.py:408-410)
        plan = []
        for i in range(S):
            t = ts[i:i + 1]
            st = dict(t_input=float((t - 1. / sch.total_N) * 1000.), sigma=float(sch.sigma(t)), alpha=float(sch.alpha(t)))
            c = (1.0, 0.0, 0.0, 0.0) if i == 0 else self._update(ts, i, 2, _tau(ts[i], eta), corrector=True)
            j = i + 1
            last = j == S
            p = self._update(ts, j, 1 if (j == 1 or last) else 2, 0 if last else _tau(ts[j], eta), corrector=False)
            st.update(zip(("c_x", "c_m0", "c_m1", "c_noise"), c))
            st.update(zip(("p_x", "p_m0", "p_m1", "p_noise"), p))
            plan.append(st)
        self._plans[key] = plan
        return plan

    # ---- device side
    def _run(self, x, x_pred, m_prev, bufs, plan, t_dev, cond, guided, cfg, model_kwargs, noise: Optional[Sequence]):
        """All S evaluations.  noise None: draw xi_1 .. xi_S from the default generator into the two `bufs`, after the
        reference's discarded draw at init (sa_solver.py:785); xi_{i+1} is drawn before evaluation i, which is the same
        stream since the denoiser draws nothing.  Otherwise `noise[i - 1]` is xi_i."""
        if noise is None:
            bufs[0].normal_()
        for i, (st, t_in) in enumerate(zip(plan, t_dev)):
            if noise is None:
                bufs[(i + 1) % 2].normal_()
                cur, nxt = bufs[i % 2], bufs[(i + 1) % 2]
            else:
                cur, nxt = (noise[i - 1] if i else None), noise[i]
            out = self.model(torch.cat([x_pred, x_pred]) if guided else x_pred, t_in, cond, **model_kwargs)
            lib.sa_solver_step(step_input(out), x, x_pred, m_prev, cur if st["c_noise"] else None,
                               nxt if st["p_noise"] else None, guided=guided, cfg_scale=cfg,
                               **{k: st[k] for k in _STEP_KEYS})
        return x_pred

    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None, img_callback=None,
               quantize_x0=False, eta=0., mask=None, x0=None, temperature=1., noise_dropout=0., score_corrector=None,
               corrector_kwargs=None, verbose=True, x_T=None, log_every_t=100, unconditional_guidance_scale=1.,
               unconditional_conditioning=None, model_kwargs={}, noise: Optional[Sequence[torch.Tensor]] = None,
               cuda_graph: bool = False, **kwargs):
        """Same signature as the reference (diffusion/sa_sampler.py:30-55) plus `noise` (the draws xi_1 .. xi_S, i.e. the
        reference's randn_like draws after the discarded one; default: drawn from the default CUDA generator exactly as the
        reference draws them) and `cuda_graph`.  Returns `(x, None)`."""
        if (mask is not None or x0 is not None or quantize_x0 or score_corrector is not None or normals_sequence is not None
                or noise_dropout != 0. or temperature != 1.):
            raise NotImplementedError("mask, x0, quantize_x0, score_corrector, normals_sequence, noise_dropout and temperature "
                                      "are not supported (scripts/inference.py passes none of them)")
        if isinstance(conditioning, dict):
            raise NotImplementedError("dict conditioning is not supported: pass the caption embedding tensor")
        if not isinstance(conditioning, torch.Tensor):
            raise ValueError("conditioning (the caption embedding) is required")
        device = x_T.device if x_T is not None else torch.device(self.device)
        guided = not (unconditional_guidance_scale == 1. or unconditional_conditioning is None)   # sa_solver.py:311-312
        if device.type != "cuda" or not conditioning.is_cuda or (guided and not unconditional_conditioning.is_cuda):
            raise RuntimeError("pixart_sigma_b200.sa_sampler has no CPU path: latents and conditioning must be CUDA tensors")
        size = (batch_size,) + tuple(shape)
        if len(size) != 4 or size[1] != 4 or (size[2] * size[3]) % 4:
            raise ValueError("shape must be (4, h, w) with h*w a multiple of 4")
        plan = self.plan(S, eta)
        if noise is not None:
            noise = [z.to(device=device, dtype=torch.float32).contiguous() for z in noise]
            if len(noise) != S or any(tuple(z.shape) != size for z in noise):
                raise ValueError(f"noise must be {S} tensors of shape {size}")
        if x_T is None:
            x_T = torch.randn(size, device=device)                       # sa_sampler.py:70-71
        elif tuple(x_T.shape) != size:
            raise ValueError(f"x_T must have shape {size}")
        cond = self._cfg_cond(unconditional_conditioning, conditioning) if guided else conditioning     # sa_solver.py:316
        cfg = float(unconditional_guidance_scale) if guided else 1.0
        rows = 2 * batch_size if guided else batch_size
        t_dev = [torch.full((rows,), st["t_input"], dtype=torch.float32, device=device) for st in plan]

        def loop(x0, k, draws):
            x = x0.to(torch.float32).contiguous().clone()
            x_pred = x.clone()
            m_prev, bufs = torch.empty_like(x), [torch.empty_like(x), torch.empty_like(x)]
            return self._run(x, x_pred, m_prev, bufs, plan[:k], t_dev[:k], cond, guided, cfg, model_kwargs, draws)
        if cuda_graph:
            # the per-evaluation scalars and t_input are baked into the captured kernel arguments
            extras = (guided, cfg, cond.data_ptr(), tuple(cond.shape),
                      tuple(tuple(st[k] for k in ("t_input",) + _STEP_KEYS) for st in plan))
            out = self._graphs.sample(self.model, model_kwargs, extras, x_T, noise, loop, (cond, t_dev))
        else:
            out = loop(x_T, None, noise)
        return out.to(x_T.dtype), None
