"""LCM on the sm_90a kernels: the few-step sampler and latent consistency distillation (PixArt-Sigma LCM recipe).

Mirrors what `train_scripts/train_pixart_lcm.py` runs with `configs/pixart_sigma_config/PixArt_sigma_xl2_img1024_lcm.py`:
  * `LCMScheduler` -- the reference's `diffusion/lcm_scheduler.py` (constructor, `set_timesteps`, `step`) for its one
    configuration: linear betas, epsilon prediction.  Options that would change the arithmetic raise `NotImplementedError`.
    `step` is one `pxa_lcm_step` launch with the scalars computed on the host by the reference's float32 torch operations.
  * `LCMSampler` -- the 4-step loop of `log_validation` (:105-135) for a batch: same results, same draws from the CPU
    generator (taken up front, one host-to-device copy per call), optionally captured into one CUDA graph.
  * `LCMDistiller` -- one consistency-distillation step (:223-303) and `ema_update` (:48-53): the student through the
    training path, the teacher as ONE forward at batch 2b over [y ; uncond], the EMA target forward, and the glue as two
    kernels (`pxa_lcm_teacher_target`, `pxa_lcm_consistency_loss`) over a 50-row coefficient table uploaded once, so a step
    never syncs the host.  `update_ema()` is one `pxa_ema_flat` launch over the fp32 EMA master (kept in the student
    reducer's bucket layout) that also writes the EMA model's bf16 weights.
  * `GraphedLCMStep` -- the whole step captured as one CUDA graph, in the manner of `training.GraphedTrainStep`.
The caller keeps `optim.clip_grad_norm_` and `optim.FlatCAME` as they are.  There is no CPU path.
"""
from __future__ import annotations

import copy
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import lib
from .sampler import _capture, _denoiser_key, _denoiser_params, _step_input
from .training import IDDPMLoss

__all__ = ["LCMScheduler", "LCMSchedulerOutput", "LCMSampler", "LCMDistiller", "GraphedLCMStep", "boundary_scalings",
           "distill_table"]


def boundary_scalings(timestep: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(c_skip, c_out) of `scalings_for_boundary_conditions` (train_pixart_lcm.py:63-67) and
    `LCMScheduler.get_scalings_for_boundary_condition_discrete` (lcm_scheduler.py:301-308): sigma_data = 0.5, t / 0.1.
    On an int64 tensor the arithmetic is float32, as in the reference."""
    c_skip = 0.5 ** 2 / ((timestep / 0.1) ** 2 + 0.5 ** 2)
    c_out = (timestep / 0.1) / ((timestep / 0.1) ** 2 + 0.5 ** 2) ** 0.5
    return c_skip, c_out


# ================================================================================================= sampler
@dataclass
class LCMSchedulerOutput:
    prev_sample: torch.Tensor
    denoised: torch.Tensor


class LCMScheduler:
    """`diffusion/lcm_scheduler.py::LCMScheduler` for linear betas and epsilon prediction (the configuration of
    `log_validation`, train_pixart_lcm.py:108).  `config` holds every constructor argument, defaults included."""

    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, clip_sample: bool = True, set_alpha_to_one: bool = True,
                 steps_offset: int = 0, prediction_type: str = "epsilon", thresholding: bool = False,
                 dynamic_thresholding_ratio: float = 0.995, clip_sample_range: float = 1.0, sample_max_value: float = 1.0,
                 timestep_spacing: str = "leading", rescale_betas_zero_snr: bool = False):
        if trained_betas is not None or beta_schedule != "linear" or rescale_betas_zero_snr:
            raise NotImplementedError("only beta_schedule='linear' without trained_betas or zero-SNR rescaling is supported")
        if prediction_type != "epsilon":
            raise NotImplementedError("only prediction_type='epsilon' is supported")
        self.config = SimpleNamespace(
            num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end, beta_schedule=beta_schedule,
            trained_betas=trained_betas, clip_sample=clip_sample, set_alpha_to_one=set_alpha_to_one, steps_offset=steps_offset,
            prediction_type=prediction_type, thresholding=thresholding, dynamic_thresholding_ratio=dynamic_thresholding_ratio,
            clip_sample_range=clip_sample_range, sample_max_value=sample_max_value, timestep_spacing=timestep_spacing,
            rescale_betas_zero_snr=rescale_betas_zero_snr)
        # float32 torch, as lcm_scheduler.py:206-214
        self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))

    def scale_model_input(self, sample: torch.Tensor, timestep: Optional[int] = None) -> torch.Tensor:
        return sample

    def set_timesteps(self, num_inference_steps: int, lcm_origin_steps: int, device=None) -> None:
        """lcm_scheduler.py:288-299: origin steps (1..lcm_origin_steps) * c - 1, every (origin // steps)-th from the end."""
        if num_inference_steps > self.config.num_train_timesteps:
            raise ValueError(f"`num_inference_steps`: {num_inference_steps} cannot be larger than `self.config.train_timesteps`:"
                             f" {self.config.num_train_timesteps}")
        self.num_inference_steps = num_inference_steps
        c = self.config.num_train_timesteps // lcm_origin_steps
        origin = np.asarray(list(range(1, lcm_origin_steps + 1))) * c - 1
        skipping_step = len(origin) // num_inference_steps
        timesteps = origin[::-skipping_step][:num_inference_steps]
        self.timesteps = torch.from_numpy(timesteps.copy()).to(device)

    def step_scalars(self, timeindex: int, timestep) -> Dict[str, float]:
        """The scalars of `pxa_lcm_step` for step `timeindex` at `timestep`, by the float32 operations of
        lcm_scheduler.py:367-401 on a 0-d int64 timestep (what the reference's loop passes)."""
        t = torch.as_tensor(int(timestep), dtype=torch.int64)
        prev_timeindex = timeindex + 1
        prev_t = self.timesteps[prev_timeindex].cpu() if prev_timeindex < len(self.timesteps) else t
        ac_t = self.alphas_cumprod[t]
        ac_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        beta_t, beta_prev = 1 - ac_t, 1 - ac_prev
        c_skip, c_out = boundary_scalings(t)
        multi = len(self.timesteps) > 1
        return dict(sqrt_alpha=float(ac_t.sqrt()), sqrt_beta=float(beta_t.sqrt()), c_skip=float(c_skip), c_out=float(c_out),
                    c_prev=float(ac_prev.sqrt()) if multi else 1.0, c_noise=float(beta_prev.sqrt()) if multi else 0.0)

    def step(self, model_output: torch.Tensor, timeindex: int, timestep, sample: torch.Tensor, eta: float = 0.0,
             use_clipped_model_output: bool = False, generator=None, variance_noise: Optional[torch.Tensor] = None,
             return_dict: bool = True):
        """One `pxa_lcm_step` launch.  With more than one timestep the noise is `torch.randn(model_output.shape)` from the
        CPU default generator, moved to the device, as the reference draws it (also on the last step)."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        if generator is not None or variance_noise is not None:
            raise NotImplementedError("generator / variance_noise are not used by the reference's step")
        if not (model_output.is_cuda and sample.is_cuda):
            raise RuntimeError("pixart_sigma_b200.lcm has no CPU path: model_output and sample must be CUDA tensors")
        st = self.step_scalars(timeindex, timestep)
        x = sample.to(torch.float32).contiguous()
        noise = None
        if len(self.timesteps) > 1:
            noise = torch.randn(model_output.shape).to(model_output.device)
        denoised, prev = torch.empty_like(x), torch.empty_like(x)
        lib.lcm_step(_step_input(model_output), x, noise, denoised, prev, **st)
        if not return_dict:
            return prev, denoised
        return LCMSchedulerOutput(prev_sample=prev, denoised=denoised)


class LCMSampler:
    """The LCM loop of `log_validation` (train_pixart_lcm.py:105-135) for a batch of n: per step
    `model_fn(x, ts, **model_kwargs)[:, :4]` at int64 ts of shape (n,), then `LCMScheduler.step`; returns the last
    `denoised` (fp32).  For `PixArtMS` pass `model_kwargs=dict(y=..., mask=..., data_info=...)`."""

    def __init__(self, model_fn: Callable, **scheduler_kwargs):
        self.model = model_fn
        self.scheduler = LCMScheduler(**scheduler_kwargs)
        self._params = _denoiser_params(model_fn)
        self._plans: Dict[tuple, List[dict]] = {}
        self._graphs: Dict[tuple, tuple] = {}

    def plan(self, steps: int, lcm_origin_steps: int = 50) -> List[dict]:
        """Per step: the int64 timestep and the scalars of `pxa_lcm_step`."""
        key = (int(steps), int(lcm_origin_steps))
        if key not in self._plans:
            sch = self.scheduler
            sch.set_timesteps(steps, lcm_origin_steps)
            self._plans[key] = [dict(t=int(t), **sch.step_scalars(i, t)) for i, t in enumerate(sch.timesteps)]
        return self._plans[key]

    @staticmethod
    def draw_noise(steps: int, shape: Sequence[int], pin: bool = False) -> Optional[torch.Tensor]:
        """The reference's CPU draws of one loop, in its order: `torch.randn(shape)` at every step when steps > 1 (the last
        one is drawn and discarded), none for a single step."""
        if steps <= 1:
            return None
        buf = torch.empty((steps,) + tuple(shape), dtype=torch.float32, pin_memory=pin)
        for i in range(steps):
            torch.randn(tuple(shape), out=buf[i])
        return buf

    def _run(self, x, denoised, plan, ts_dev, noise, model_kwargs):
        for i, (st, ts) in enumerate(zip(plan, ts_dev)):
            out = self.model(x, ts, **model_kwargs)
            lib.lcm_step(_step_input(out[:, :4]), x, noise[i] if st["c_noise"] != 0.0 else None, denoised, x,
                         **{k: st[k] for k in ("sqrt_alpha", "sqrt_beta", "c_skip", "c_out", "c_prev", "c_noise")})
        return denoised

    @torch.no_grad()
    def sample(self, x_T: torch.Tensor, steps: int = 4, lcm_origin_steps: int = 50, model_kwargs: Optional[dict] = None,
               noise: Optional[torch.Tensor] = None, cuda_graph: bool = False) -> torch.Tensor:
        """x_T (n, 4, h, w) on the device.  `noise`: replays given draws (steps, n, 4, h, w) instead of drawing from the CPU
        generator; default: drawn up front in the reference's order and copied to the device once."""
        model_kwargs = dict(model_kwargs or {})
        if not x_T.is_cuda:
            raise RuntimeError("pixart_sigma_b200.lcm has no CPU path: x_T must be a CUDA tensor")
        if x_T.dim() != 4 or x_T.shape[1] != 4 or (x_T.shape[2] * x_T.shape[3]) % 4:
            raise ValueError("x_T must be (n, 4, h, w) latents with h*w a multiple of 4")
        if steps < 1:
            raise ValueError("steps must be >= 1")
        plan = self.plan(steps, lcm_origin_steps)
        shape = tuple(x_T.shape)
        if noise is None:
            host = self.draw_noise(steps, shape, pin=True)
            noise = None if host is None else host.to(x_T.device, non_blocking=True)
        elif steps > 1:
            noise = torch.as_tensor(noise)
            if tuple(noise.shape) != (steps,) + shape:
                raise ValueError(f"noise must have shape {(steps,) + shape}")
            noise = noise.to(device=x_T.device, dtype=torch.float32).contiguous()
        else:
            noise = None
        n = shape[0]
        ts_dev = [torch.full((n,), st["t"], dtype=torch.int64, device=x_T.device) for st in plan]
        if cuda_graph:
            return self._sample_graphed(x_T, plan, ts_dev, noise, model_kwargs)
        x = x_T.to(torch.float32).contiguous().clone()
        return self._run(x, torch.empty_like(x), plan, ts_dev, noise, model_kwargs)

    def _sample_graphed(self, x_T, plan, ts_dev, noise, model_kwargs):
        # the step scalars and timesteps are baked into the captured launches, model_kwargs tensors and the parameters
        # (through derived weight copies) into the captured forward: all are part of the key
        kw_id, wkey = _denoiser_key(self.model, self._params, model_kwargs)
        key = (tuple(x_T.shape), x_T.device.index, kw_id, wkey, tuple(tuple(sorted(st.items())) for st in plan))
        if key not in self._graphs:
            z_in = torch.empty(x_T.shape, dtype=torch.float32, device=x_T.device)
            x, den = torch.empty_like(z_in), torch.empty_like(z_in)
            noise_in = None if noise is None else torch.zeros_like(noise)

            def warmup():
                x.copy_(x_T)
                self._run(x, den, plan[:2], ts_dev[:2], noise_in, model_kwargs)

            def body():
                x.copy_(z_in)
                self._run(x, den, plan, ts_dev, noise_in, model_kwargs)
            graph = _capture(warmup, body)
            self._graphs[key] = (graph, z_in, den, noise_in, ts_dev)
        graph, z_in, den, noise_in = self._graphs[key][:4]
        z_in.copy_(x_T)
        if noise_in is not None:
            noise_in.copy_(noise)
        graph.replay()
        return den.clone()


# ================================================================================================= distillation
def distill_table(num_ddim_timesteps: int = 50, num_train_timesteps: int = 1000):
    """Host plan of the distillation step.  Returns (ddim_timesteps int64 [N], alpha_cumprods_prev fp64 [N], rows) with one
    row per DDIM index: the fields of `PxaLcmRow` (include/pixart_sm100.h), each computed by the reference's own
    operations -- IDDPM's fp64 tables indexed and rounded to fp32 (`_extract_into_tensor`), the float32 boundary scalings on
    int64 timesteps, and `DDIMSolver` (train_pixart_lcm.py:76-101) in fp64."""
    T, N = num_train_timesteps, num_ddim_timesteps
    tab = IDDPMLoss(T).tab
    ac = np.cumprod(1.0 - np.linspace(1000 / T * 0.0001, 1000 / T * 0.02, T, dtype=np.float64))
    ddim_ts = (np.arange(1, N + 1) * (T // N)).round().astype(np.int64) - 1
    acp_prev = torch.from_numpy(np.asarray([ac[0]] + ac[ddim_ts[:-1]].tolist()))
    topk = T // N
    f32 = lambda name, t: float(torch.from_numpy(tab[name])[t].float())
    rows = []
    for k in range(N):
        s = torch.tensor(int(ddim_ts[k]), dtype=torch.int64)
        t = torch.where(s - topk < 0, torch.zeros_like(s), s - topk)
        cs_s, co_s = boundary_scalings(s)
        cs_t, co_t = boundary_scalings(t)
        rows.append(dict(sra_s=f32("sqrt_recip_ac", s), srm1_s=f32("sqrt_recipm1_ac", s), cskip_s=float(cs_s), cout_s=float(co_s),
                         sra_t=f32("sqrt_recip_ac", t), srm1_t=f32("sqrt_recipm1_ac", t), cskip_t=float(cs_t), cout_t=float(co_t),
                         sqrt_acp=float(acp_prev[k].sqrt()), sqrt_1macp=float((1.0 - acp_prev[k]).sqrt())))
    return torch.from_numpy(ddim_ts), acp_prev, rows


def _upload(struct_array, device) -> torch.Tensor:
    return torch.frombuffer(bytearray(bytes(struct_array)), dtype=torch.uint8).to(device)


def _inference_copy(model: torch.nn.Module) -> torch.nn.Module:
    """A no-grad eval copy of `model` with bf16 parameters (buffers keep their dtype) and its own workspace."""
    from . import autograd as ag
    from .model import _Workspace
    m = copy.deepcopy(model)
    ag.clear_shadow_cache(m)
    for mod in m.modules():
        if "_ln_fusion" in mod.__dict__:
            mod.__dict__["_ln_fusion"] = None
        if "_kv_batch" in mod.__dict__:
            mod.__dict__["_kv_batch"] = None
        if isinstance(getattr(mod, "_ws", None), _Workspace):
            mod._ws = _Workspace()
    for p in m.parameters():
        p.requires_grad_(False)
        if p.dtype != torch.bfloat16:
            p.data = p.data.to(torch.bfloat16)
    m.eval()
    if hasattr(m, "output_dtype"):
        m.output_dtype = torch.float32           # the final linear is fp32: keep its output unrounded
    return m


def _check_ema_forward(ema: torch.nn.Module) -> None:
    """The EMA model's weights are rewritten by a kernel, which does not bump `_version`: the forward modes that keep
    copies derived from the weights and keyed on `_version` (fused LayerNorm-modulate, batched kv_linear) would go stale."""
    from . import model as _m
    if getattr(ema, "fuse_ln_modulate", False) or (_m._KV_BATCH and len(getattr(ema, "blocks", ())) > 1):
        raise RuntimeError("LCMDistiller: the EMA model cannot use fuse_ln_modulate or PXA_KV_BATCH=1 (their derived weight "
                           "copies are keyed on _version, which pxa_ema_flat does not bump)")


class _ConsistencyLoss(torch.autograd.Function):
    """mean consistency loss over `pxa_lcm_consistency_loss`; the gradient with respect to the student's output is written
    by the same launch."""

    @staticmethod
    def forward(ctx, student_out, ema_out, x_t, x_prev, index, table, partials, loss_type, huber_c):
        d = torch.empty(student_out.shape, dtype=torch.float32, device=student_out.device)
        loss = torch.empty((), dtype=torch.float32, device=student_out.device)
        lib.lcm_consistency_loss(student_out, ema_out, x_t, x_prev, index, table, d, loss, partials, loss_type=loss_type,
                                 huber_c=huber_c)
        ctx.save_for_backward(d)
        return loss

    @staticmethod
    def backward(ctx, grad):
        (d,) = ctx.saved_tensors
        return d * grad, None, None, None, None, None, None, None, None


def _dup(v):
    return torch.cat([v, v]) if isinstance(v, torch.Tensor) else v


class LCMDistiller:
    """Latent consistency distillation (train_pixart_lcm.py:223-309) on the native kernels; see the module docstring.

    student: the online model (fp32 master parameters, train mode) whose gradients `reducer` (parallel.GradBucketReducer)
    buckets; the reducer's parameters are flattened here.  teacher / ema: default bf16 copies of the student.  A given
    `ema` is initialised from its own values and its parameters become bf16 views of the EMA's shadow buckets.  The EMA's
    fp32 master lives in the reducer's bucket layout; `ema_state_dict()` returns it under the model's key names.
    `w` is the guidance scale of the teacher's CFG (config `cfg_scale`)."""

    def __init__(self, student: torch.nn.Module, reducer, teacher: Optional[torch.nn.Module] = None,
                 ema: Optional[torch.nn.Module] = None, w: float = 4.5, loss_type: str = "huber", huber_c: float = 1e-3,
                 ema_decay: float = 0.95, num_ddim_timesteps: int = 50, num_train_timesteps: int = 1000):
        if loss_type not in ("huber", "l2"):
            raise NotImplementedError("loss_type must be 'huber' or 'l2' (train_pixart_lcm.py:295-298)")
        if loss_type == "huber" and not huber_c > 0:
            raise ValueError("huber_c must be positive")
        if not 0.0 <= ema_decay <= 1.0:
            raise ValueError("ema_decay must be in [0, 1]")
        if not 0 < num_ddim_timesteps <= min(num_train_timesteps, lib.LCM_MAX_ROWS):
            raise ValueError(f"num_ddim_timesteps must be in 1..{min(num_train_timesteps, lib.LCM_MAX_ROWS)}")
        self.student, self.reducer = student, reducer
        self.w, self.huber_c, self.ema_decay = float(w), float(huber_c), float(ema_decay)
        self.loss_type = lib.LCM_HUBER if loss_type == "huber" else lib.LCM_L2
        reducer.flatten_params()
        flats = [b["flat_param"] for b in reducer.buckets]
        if any(not f.is_cuda or f.dtype != torch.float32 for f in flats):
            raise RuntimeError("LCMDistiller: the student's reducer must hold fp32 CUDA parameters (use model.float().cuda())")
        dev = flats[0].device
        self.device = dev
        self.loss_fn = IDDPMLoss(num_train_timesteps)
        ddim_ts, _, rows = distill_table(num_ddim_timesteps, num_train_timesteps)
        self.rows = rows
        self.topk = num_train_timesteps // num_ddim_timesteps
        self.num_ddim_timesteps = num_ddim_timesteps
        self.ddim_timesteps = ddim_ts.to(dev)
        self.table = _upload((lib.LcmRow * len(rows))(*[lib.LcmRow(**r) for r in rows]), dev)       # uploaded once
        self.partials = torch.empty(lib.LCM_LOSS_PARTS, dtype=torch.float64, device=dev)
        self.uncond = student.y_embedder.y_embedding.detach().clone()     # train_pixart_lcm.py:191 (fixed at start)
        self.teacher = teacher if teacher is not None else _inference_copy(student)
        self.teacher.requires_grad_(False)
        self._build_ema(ema)

    # ---- EMA: fp32 master + bf16 forward weights, both in the reducer's bucket layout
    def _build_ema(self, ema):
        names = {id(p): n for n, p in self.student.named_parameters()}
        given = ema is not None
        self.ema = ema if given else _inference_copy(self.student)
        self.ema.requires_grad_(False)
        ema_params = dict(self.ema.named_parameters())
        self.master, self.shadow, self.layout = [], [], []
        entries = []
        with torch.no_grad():
            for b in self.reducer.buckets:
                fp = b["flat_param"]
                master = torch.zeros_like(fp)
                shadow = torch.zeros(fp.numel(), dtype=torch.bfloat16, device=fp.device)
                off, layout = 0, []
                for p in b["params"]:
                    name, n = names[id(p)], p.numel()
                    e = ema_params.get(name)
                    if e is None or e.shape != p.shape:
                        raise ValueError(f"LCMDistiller: the EMA model has no parameter {name!r} of shape {tuple(p.shape)}")
                    master[off: off + n].copy_((e if given else p).detach().reshape(-1))
                    layout.append((name, off, p.shape))
                    off += n
                shadow[:off].copy_(master[:off])
                for name, o, shape in layout:
                    ema_params[name].data = shadow[o: o + int(np.prod(shape))].view(shape)
                self.master.append(master)
                self.shadow.append(shadow)
                self.layout.append(layout)
                entries.append(lib.EmaBucket(master=master.data_ptr(), src=fp.data_ptr(), shadow=shadow.data_ptr(), n=off))
            for e in self.ema.parameters():                   # parameters outside the buckets: plain bf16 copies
                if e.dtype != torch.bfloat16:
                    e.data = e.data.to(torch.bfloat16)
        self._ema_n = [e.n for e in entries]
        self._ema_table = _upload((lib.EmaBucket * len(entries))(*entries), self.device)
        _check_ema_forward(self.ema)

    @torch.no_grad()
    def update_ema(self) -> None:
        """`ema_update(model_ema, model, ema_decay)` (train_pixart_lcm.py:48-53) in one launch: fp32 master and the EMA
        model's bf16 weights.  The student's parameters must still be the reducer's flat buckets."""
        self.reducer.flatten_params()
        lib.ema_flat(self._ema_table, n_buckets=len(self._ema_n), max_n=max(self._ema_n), rate=self.ema_decay)

    def ema_state_dict(self) -> Dict[str, torch.Tensor]:
        """The EMA model's state dict with every bucketed parameter as its fp32 master value (what `save_checkpoint(model_ema=
        ...)` stores as `state_dict_ema`); buffers as the EMA model holds them."""
        sd = {k: v.detach().clone() for k, v in self.ema.state_dict().items()}
        for master, layout in zip(self.master, self.layout):
            for name, off, shape in layout:
                sd[name] = master[off: off + int(np.prod(shape))].view(shape).clone()
        return sd

    # ---- one distillation step
    def draw(self, latents: torch.Tensor):
        """The step's random inputs in the reference's order (train_pixart_lcm.py:233-238): noise, then the DDIM indices,
        both from the device generator."""
        noise = torch.randn_like(latents)
        index = torch.randint(0, self.num_ddim_timesteps, (latents.shape[0],), device=latents.device).long()
        return noise, index

    def _forward_loss(self, latents, y, mask, data_info, noise, index) -> torch.Tensor:
        from . import autograd as ag
        b = latents.shape[0]
        start = self.ddim_timesteps[index]
        t = (start - self.topk).clamp_min(0)
        x_t = self.loss_fn.q_sample(latents, start, noise).contiguous()
        ag.refresh_shadows(self.student)
        out_s = self.student(x_t, start, y, mask=mask, data_info=data_info)
        if out_s.dtype != torch.float32:
            out_s = out_s.float()
        with torch.no_grad():
            uncond = self.uncond.to(device=y.device, dtype=y.dtype).expand(b, 1, *self.uncond.shape)
            m2 = mask if mask is None or mask.shape[0] != b else torch.cat([mask, mask])
            di2 = None if data_info is None else {k: _dup(v) if isinstance(v, torch.Tensor) and v.shape[0] == b else v
                                                  for k, v in data_info.items()}
            out_t = self.teacher(torch.cat([x_t, x_t]), torch.cat([start, start]), torch.cat([y, uncond]), mask=m2, data_info=di2)
            x_prev = torch.empty_like(x_t)
            lib.lcm_teacher_target(_step_input(out_t), x_t, index, self.table, x_prev, w=self.w)
            _check_ema_forward(self.ema)
            out_e = self.ema(x_prev, t, y, mask=mask, data_info=data_info)
        return _ConsistencyLoss.apply(out_s, _step_input(out_e), x_t, x_prev, index, self.table, self.partials, self.loss_type,
                                      self.huber_c)

    def step(self, latents: torch.Tensor, y: torch.Tensor, mask: Optional[torch.Tensor] = None, data_info=None,
             noise: Optional[torch.Tensor] = None, index: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Steps 1-7 of train_pixart_lcm.py:232-301 plus the backward: returns the loss as a 0-d device tensor (no host
        sync) with the student's gradients accumulated into the reducer's buckets (call `reducer.zero_grad()` first).
        noise / index: given draws (default: `draw(latents)`)."""
        if not latents.is_cuda or latents.dim() != 4 or latents.shape[1] != 4:
            raise ValueError("latents must be (b, 4, h, w) CUDA tensors")
        latents = latents.to(torch.float32)
        if noise is None or index is None:
            dn, di = self.draw(latents)
            noise = dn if noise is None else noise
            index = di if index is None else index
        index = index.to(device=latents.device, dtype=torch.int64).contiguous()
        self.reducer.start()
        loss = self._forward_loss(latents, y, mask, data_info, noise, index)
        loss.backward()
        self.reducer.finish()
        return loss.detach()


class GraphedLCMStep:
    """One distillation step captured as ONE CUDA graph, in the manner of `training.GraphedTrainStep`: gradient zeroing, the
    student / teacher / EMA forwards, the loss and the backward; with `optimizer_step` (e.g. `lambda: (clip_grad_norm_(
    reducer, 0.01), came.step())`) also that call and then the EMA update, so one replay is one whole step of the
    reference.  Without it the caller runs clip, the optimizer and `distiller.update_ema()` after each replay.

    Static inputs (latents, y, mask, noise, index) are copied in per call; shapes are fixed per instance.  Host-side
    bookkeeping inside `optimizer_step` (e.g. FlatCAME's step counter) runs at capture only.  Single process only.
    No autograd graph through the student may be alive while the step is built (e.g. an eager loss kept for logging): its
    parameters' cached gradient accumulators keep the stream they were created on, and a captured backward that reuses them
    would have to synchronise with that stream."""

    def __init__(self, distiller: LCMDistiller, example: Sequence[Optional[torch.Tensor]],
                 optimizer_step: Optional[Callable[[], None]] = None, warmup: int = 2):
        if distiller.reducer.world > 1:
            raise NotImplementedError("GraphedLCMStep captures a single-process step (no collectives)")
        self.d = distiller
        dev = distiller.device
        self.static = [None if v is None else torch.empty_like(v, device=dev) for v in example]
        self._copy_in(example)
        lat, y, mask, noise, index = self.static
        di = None

        def fwd_bwd():
            distiller.reducer.zero_grad()
            loss = distiller._forward_loss(lat, y, mask, di, noise, index)
            loss.backward()
            return loss.detach()

        def full():
            loss = fwd_bwd()
            if optimizer_step is not None:
                optimizer_step()
                distiller.update_ema()
            return loss

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(warmup):                       # forward / backward only: the optimizer and the EMA keep their state
                fwd_bwd()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        distiller.reducer.start()
        with torch.cuda.graph(self.graph):
            self.loss = full()

    def _copy_in(self, batch):
        for dst, src in zip(self.static, batch):
            if dst is not None:
                dst.copy_(src, non_blocking=True)

    def __call__(self, latents, y, mask, noise, index) -> torch.Tensor:
        self._copy_in((latents, y, mask, noise, index))
        self.d.reducer.start()
        self.graph.replay()
        return self.loss
