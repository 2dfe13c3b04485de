"""IDDPM ancestral sampling loop around the denoiser -- the third caller of the path in `scripts/inference.py`
(`--sampling_algo iddpm`, inference.py:89-102: `IDDPM(str(sample_steps)).p_sample_loop(model.forward_with_cfg, z.shape, z,
clip_denoised=False, model_kwargs=..., device=...)`), next to the DPM-Solver++ loop (`sampler.py`), the SA-Solver loop
(`sa_sampler.py`) and the training loss (`training.py`).  A restatement of

    diffusion/iddpm.py:10-53              IDDPM(...) factory (linear betas, learned-range variance, epsilon prediction)
    diffusion/model/respace.py:12-94      space_timesteps / SpacedDiffusion (re-derived betas, timestep map)
    diffusion/model/respace.py:121-134    _WrappedModel (the model sees the ORIGINAL timestep index, as `timestep=`)
    diffusion/model/gaussian_diffusion.py:280-361, 405-446, 493-540   p_mean_variance / p_sample / p_sample_loop_progressive

so that sampling runs without the reference package; `install_into_reference()` re-points `diffusion.IDDPM` here.

`p_sample_loop` on CUDA latents is the native loop:
  * every per-step scalar is read once on the host from the fp64 tables and rounded to fp32 exactly as `_extract_into_tensor`
    rounds it, and the mapped timesteps of all steps are uploaded once, so a step never copies to or syncs with the host;
  * the CFG mix of `forward_with_cfg` (channels 0..2 only, as the reference), the learned-range variance, pred_x0, the
    posterior mean, the noise term and the next model input are ONE elementwise sm_90a kernel per step (`pxa_iddpm_step`,
    include/pixart_sm100.h).  When the model is the bound `forward_with_cfg` of this package's `PixArtMS` / `PixArt`, the loop
    calls its `forward` on the [img[:n] ; img[:n]] batch the kernel wrote and mixes in the kernel; any other callable is
    called as `_WrappedModel` calls it and its output is used as it is;
  * each step draws `randn_like(img)` from the default generator of the latents' device, the last step included, so a seeded
    run consumes the reference loop's random numbers; `noise_draws=` replays given draws instead;
  * `cuda_graph=True` captures the whole loop -- every forward, draw and step kernel -- into one CUDA graph.
On CPU latents `p_sample_loop` runs the elementwise torch restatement (`p_sample_loop_progressive`, which is also the
per-step generator on any device), pinned against the unmodified reference sampler by `tests/golden/iddpm_sample_*.pt`.
"""
from __future__ import annotations

from typing import Callable, Dict, Iterator, List, Optional, Sequence

import numpy as np
import torch

from . import lib
from .capture import CapturedLoops, step_input
from .model import PixArt, PixArtMS

# pxa_iddpm_step scalar -> IDDPMSampler.tab entry it is read from (p_mean_variance's _extract_into_tensor calls)
_STEP_TABLES = (("sqrt_recip_ac", "sqrt_recip_ac"), ("sqrt_recipm1_ac", "sqrt_recipm1_ac"), ("post_c1", "post_c1"),
                ("post_c2", "post_c2"), ("log_beta", "log_betas"), ("post_logvar", "post_logvar"))
_STEP_KEYS = tuple(k for k, _ in _STEP_TABLES)


def space_timesteps(num_timesteps: int, section_counts) -> List[int]:
    """Timesteps of the original process kept by a respacing string such as "100" or "10,15,20" (respace.py:12-63)."""
    if isinstance(section_counts, str):
        if section_counts.startswith("ddim"):
            want = int(section_counts[len("ddim"):])
            for i in range(1, num_timesteps):
                if len(range(0, num_timesteps, i)) == want:
                    return sorted(range(0, num_timesteps, i))
            raise ValueError(f"cannot create exactly {num_timesteps} steps with an integer stride")
        section_counts = [int(x) for x in section_counts.split(",")]
    size_per, extra = divmod(num_timesteps, len(section_counts))
    start, steps = 0, []
    for i, count in enumerate(section_counts):
        size = size_per + (1 if i < extra else 0)
        if size < count:
            raise ValueError(f"cannot divide section of {size} steps into {count}")
        stride = 1 if count <= 1 else (size - 1) / (count - 1)
        cur = 0.0
        for _ in range(count):
            steps.append(start + round(cur))
            cur += stride
        start += size
    return sorted(set(steps))


class IDDPMSampler:
    """`IDDPM(timestep_respacing)` restricted to what inference uses: linear schedule, epsilon prediction, learned-range
    variance (`learn_sigma=True, pred_sigma=True`)."""

    def __init__(self, timestep_respacing, diffusion_steps: int = 1000):
        scale = 1000 / diffusion_steps                                        # gaussian_diffusion.py:107-116
        base_betas = np.linspace(scale * 0.0001, scale * 0.02, diffusion_steps, dtype=np.float64)
        base_ac = np.cumprod(1.0 - base_betas, axis=0)
        if timestep_respacing is None or timestep_respacing == "":
            timestep_respacing = [diffusion_steps]
        keep = set(space_timesteps(diffusion_steps, timestep_respacing))
        self.timestep_map, betas, last = [], [], 1.0                          # respace.py:73-86
        for i, ac in enumerate(base_ac):
            if i in keep:
                betas.append(1 - ac / last)
                last = ac
                self.timestep_map.append(i)
        betas = np.array(betas, dtype=np.float64)
        self.num_timesteps = len(betas)
        alphas = 1.0 - betas
        ac = np.cumprod(alphas, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        post_var = betas * (1.0 - ac_prev) / (1.0 - ac)                       # gaussian_diffusion.py:214-227
        self.tab = {
            "sqrt_recip_ac": np.sqrt(1.0 / ac), "sqrt_recipm1_ac": np.sqrt(1.0 / ac - 1),
            "post_logvar": np.log(np.append(post_var[1], post_var[1:])) if len(post_var) > 1 else np.array([]),
            "post_c1": betas * np.sqrt(ac_prev) / (1.0 - ac), "post_c2": (1.0 - ac_prev) * np.sqrt(alphas) / (1.0 - ac),
            "log_betas": np.log(betas),
        }
        self._dev: Dict[str, torch.Tensor] = {}
        self._plan: Optional[List[dict]] = None
        self._tmaps: Dict[tuple, torch.Tensor] = {}
        self._graphs = CapturedLoops()

    last_capture_s = property(lambda self: self._graphs.last_capture_s)    # wall time of the latest CUDA-graph capture

    def _x(self, name: str, t: torch.Tensor) -> torch.Tensor:                 # _extract_into_tensor, :1029-1041
        key = f"{name}@{t.device}"
        if key not in self._dev:
            self._dev[key] = torch.from_numpy(self.tab[name]).to(t.device)
        return self._dev[key][t].float()[:, None, None, None]

    def p_mean_variance(self, model, x, t, clip_denoised: bool = True, model_kwargs: Optional[dict] = None):
        """:280-361 with ModelVarType.LEARNED_RANGE and ModelMeanType.EPSILON; the model is called like _WrappedModel does."""
        n, C = x.shape[:2]
        map_t = torch.tensor(self.timestep_map, device=t.device, dtype=t.dtype)[t]
        out = model(x, timestep=map_t, **(model_kwargs or {}))
        assert out.shape == (n, 2 * C, *x.shape[2:])
        eps, var_values = torch.split(out, C, dim=1)
        min_log, max_log = self._x("post_logvar", t), self._x("log_betas", t)
        frac = (var_values + 1) / 2
        log_variance = frac * max_log + (1 - frac) * min_log
        pred_xstart = self._x("sqrt_recip_ac", t) * x - self._x("sqrt_recipm1_ac", t) * eps
        if clip_denoised:
            pred_xstart = pred_xstart.clamp(-1, 1)
        mean = self._x("post_c1", t) * pred_xstart + self._x("post_c2", t) * x
        return {"mean": mean, "variance": torch.exp(log_variance), "log_variance": log_variance, "pred_xstart": pred_xstart}

    def p_sample(self, model, x, t, clip_denoised: bool = True, model_kwargs: Optional[dict] = None):
        """:405-446: x_{t-1} = mean + [t != 0] * exp(0.5 * log_variance) * noise."""
        out = self.p_mean_variance(model, x, t, clip_denoised=clip_denoised, model_kwargs=model_kwargs)
        noise = torch.randn_like(x)
        nonzero = (t != 0).float().view(-1, 1, 1, 1)
        return {"sample": out["mean"] + nonzero * torch.exp(0.5 * out["log_variance"]) * noise, "pred_xstart": out["pred_xstart"]}

    @torch.no_grad()
    def p_sample_loop_progressive(self, model, shape: Sequence[int], noise=None, clip_denoised: bool = True,
                                  model_kwargs: Optional[dict] = None, device=None, progress: bool = False) -> Iterator[dict]:
        if device is None:
            device = next(model.parameters()).device
        img = noise if noise is not None else torch.randn(*shape, device=device)
        for i in reversed(range(self.num_timesteps)):                          # :519-540
            t = torch.tensor([i] * shape[0], device=device)
            out = self.p_sample(model, img, t, clip_denoised=clip_denoised, model_kwargs=model_kwargs)
            yield out
            img = out["sample"]

    @torch.no_grad()
    def p_sample_loop(self, model, shape, noise=None, clip_denoised: bool = True, denoised_fn=None, cond_fn=None,
                      model_kwargs: Optional[dict] = None, device=None, progress: bool = False, *,
                      noise_draws: Optional[Sequence[torch.Tensor]] = None, cuda_graph: bool = False) -> torch.Tensor:
        """Same call signature as gaussian_diffusion.py:448-491 (denoised_fn / cond_fn are not used by inference.py and
        must be None; `progress` is ignored) plus two keywords of the native loop: `noise_draws`, the per-step
        `randn_like(img)` draws in the order the loop makes them (first step first, the last step's included) to replay a
        run, and `cuda_graph`, which runs the loop as one captured CUDA graph (each replay draws fresh noise).  CUDA latents
        take the native loop, CPU latents the torch restatement.  Both run without autograd, as the reference loop does, so
        the model takes its inference forward whatever the caller's grad mode."""
        if denoised_fn is not None or cond_fn is not None:
            raise NotImplementedError("denoised_fn / cond_fn are not supported by the H100 IDDPM sampling loop")
        where = noise.device if noise is not None else torch.device(device if device is not None else
                                                                    next(model.parameters()).device)
        if where.type == "cuda":
            return self._sample_native(model, shape, noise, clip_denoised, model_kwargs, where, noise_draws, cuda_graph)
        if noise_draws is not None or cuda_graph:
            raise NotImplementedError("noise_draws and cuda_graph belong to the native loop: the latents must be CUDA tensors")
        final = None
        for final in self.p_sample_loop_progressive(model, shape, noise=noise, clip_denoised=clip_denoised,
                                                    model_kwargs=model_kwargs, device=device, progress=progress):
            pass
        return final["sample"]

    def training_losses(self, *args, **kwargs):
        """Not provided: this object samples only.  A training script that does `from diffusion import IDDPM`
        (train_scripts/train.py:23, :410) must import it before `install_into_reference()`, or train with
        `pixart_sigma_b200.training.IDDPMLoss`."""
        raise NotImplementedError("pixart_sigma_b200.iddpm.IDDPM samples only (p_sample_loop): for training losses import "
                                  "diffusion.IDDPM before install_into_reference(), or use "
                                  "pixart_sigma_b200.training.IDDPMLoss")

    # ---- native loop: host side
    def plan(self) -> List[dict]:
        """One entry per step, in sampling order (t = num_timesteps - 1 down to 0): `t`, the mapped timestep `map_t` the
        model sees, and the pxa_iddpm_step scalars -- the fp64 table entries at t rounded to fp32, which is what
        `_x(name, t)` gives (`tab[name][t].float()`)."""
        if self._plan is None:
            if self.num_timesteps < 2:
                raise ValueError("the learned-range variance needs at least two sampling steps")
            self._plan = [dict(t=i, map_t=int(self.timestep_map[i]),
                               **{k: float(np.float32(self.tab[name][i])) for k, name in _STEP_TABLES})
                          for i in reversed(range(self.num_timesteps))]
        return self._plan

    def _timesteps(self, device: torch.device, rows: int) -> torch.Tensor:
        """(steps, rows) int64 mapped timesteps of every step on `device`: one upload, kept for later calls."""
        key = (str(device), rows)
        if key not in self._tmaps:
            tab = torch.tensor([[st["map_t"]] * rows for st in self.plan()], dtype=torch.int64)
            # through pinned memory: the upload does not wait for the device
            self._tmaps[key] = tab.pin_memory().to(device, non_blocking=True) if device.type == "cuda" else tab.to(device)
        return self._tmaps[key]

    # ---- native loop: device side
    def _sample_native(self, model, shape, noise, clip, model_kwargs, device, noise_draws, cuda_graph):
        size = tuple(int(v) for v in shape)
        if len(size) != 4 or size[1] != 4:
            raise ValueError(f"shape must be (N, 4, h, w), got {size}")
        plan = self.plan()
        owner = _native_cfg_owner(model)
        guided = owner is not None
        if guided and size[0] % 2:
            raise ValueError("forward_with_cfg samples CFG pairs: the batch must be [cond (n) ; uncond (n)]")
        fwd, cfg = _denoiser(model, owner, model_kwargs)
        if noise_draws is not None:
            noise_draws = [z.to(device=device, dtype=torch.float32).contiguous() for z in noise_draws]
            if len(noise_draws) != len(plan) or any(tuple(z.shape) != size for z in noise_draws):
                raise ValueError(f"noise_draws must be {len(plan)} tensors of shape {size}")
        x_T = noise if noise is not None else torch.randn(*shape, device=device)       # p_sample_loop_progressive :514-517
        if tuple(x_T.shape) != size:
            raise ValueError(f"noise must have shape {size}")
        t_all = self._timesteps(device, size[0])

        def loop(x0, k, draws):
            img = x0.to(torch.float32).contiguous().clone()
            inp = _first_input(img) if guided else None
            zbuf = torch.empty_like(img) if draws is None else None
            return self._run(fwd, img, inp, zbuf, plan[:k], t_all[:k], guided, cfg, clip, draws)
        if cuda_graph:
            extras = (guided, cfg, bool(clip), tuple(st["map_t"] for st in plan))
            return self._graphs.sample(model, model_kwargs, extras, x_T, noise_draws, loop, (t_all,))
        return loop(x_T, None, noise_draws)

    @staticmethod
    def _run(fwd, img, inp, zbuf, plan, t_all, guided, cfg, clip, draws):
        """All steps, in place on img (and, guided, on the model input inp).  draws None: each step draws into zbuf from the
        default generator after its forward, as p_sample draws after p_mean_variance; otherwise draws[k] is step k's."""
        N, C, h, w = img.shape
        for k, st in enumerate(plan):
            out = fwd(inp if guided else img, t_all[k])
            if tuple(out.shape) != (N, 2 * C, h, w):
                raise ValueError(f"the model returned {tuple(out.shape)}, expected {(N, 2 * C, h, w)} (eps and learned variance)")
            out = step_input(out, fp16=True)
            if draws is None:
                zbuf.normal_()
                z = zbuf
            else:
                z = draws[k]
            lib.iddpm_step(out, img, z if st["t"] != 0 else None, inp, guided=guided, clip=clip, cfg_scale=cfg,
                           **{key: st[key] for key in _STEP_KEYS})
        return img


def _native_cfg_owner(model: Callable) -> Optional[PixArtMS]:
    """The PixArtMS / PixArt whose own `forward_with_cfg` `model` is bound to, else None."""
    owner, fn = getattr(model, "__self__", None), getattr(model, "__func__", None)
    if isinstance(owner, PixArtMS) and fn is type(owner).forward_with_cfg and fn in (PixArtMS.forward_with_cfg,
                                                                                      PixArt.forward_with_cfg):
        return owner
    return None


def _denoiser(model: Callable, owner: Optional[PixArtMS], model_kwargs: Optional[dict]):
    """(fwd(x, t) -> learn-sigma output, cfg_scale).  Guided: the owner's forward on the 2n batch with forward_with_cfg's
    arguments, the mix left to the step kernel; otherwise `model(x, timestep=t, **model_kwargs)` (respace.py:121-134)."""
    kw = dict(model_kwargs or {})
    if owner is None:
        return (lambda x, t: model(x, timestep=t, **kw)), 1.0
    y, cfg = kw.pop("y"), float(kw.pop("cfg_scale"))
    mask, data_info = kw.pop("mask", None), kw.pop("data_info", None)
    if isinstance(owner, PixArt):                          # PixArt.forward_with_cfg passes neither data_info nor extra kwargs
        return (lambda x, t: owner.forward(x, t, y, mask)), cfg
    return (lambda x, t: owner.forward(x, t, y, mask, data_info=data_info, **kw)), cfg


def _first_input(img: torch.Tensor) -> torch.Tensor:
    half = img[: img.shape[0] // 2]
    return torch.cat([half, half]).contiguous()


def IDDPM(timestep_respacing, noise_schedule: str = "linear", use_kl: bool = False, sigma_small: bool = False,
          predict_xstart: bool = False, learn_sigma: bool = True, pred_sigma: bool = True, rescale_learned_sigmas: bool = False,
          diffusion_steps: int = 1000, snr: bool = False, return_startx: bool = False) -> IDDPMSampler:
    """Factory with the reference's signature (diffusion/iddpm.py:10-22); only the configuration inference uses exists."""
    if (noise_schedule != "linear" or use_kl or sigma_small or predict_xstart or not learn_sigma or not pred_sigma or
            rescale_learned_sigmas or snr or return_startx):
        raise NotImplementedError("only IDDPM(str(steps)) with its defaults (linear schedule, epsilon prediction, learned-range "
                                  "variance) is restated here")
    return IDDPMSampler(timestep_respacing, diffusion_steps)
