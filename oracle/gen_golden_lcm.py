"""TEST INFRASTRUCTURE ONLY -- generate tests/golden/lcm_*.pt by running the UNMODIFIED reference LCM code from the
reference checkout that oracle/refshim.py locates:

  * `diffusion/lcm_scheduler.py::LCMScheduler` (imported as is; when `diffusers` is not installed a minimal stand-in of
    `ConfigMixin`, `SchedulerMixin`, `BaseOutput` and `register_to_config` is installed first -- `register_to_config` fills
    `self.config` with every constructor argument, defaults included, which is all the scheduler reads);
  * `DDIMSolver`, `scalings_for_boundary_conditions`, `extract_into_tensor`, `append_dims` and `ema_update`, taken from
    `train_scripts/train_pixart_lcm.py` by parsing the file and executing just those top-level definitions (the script's
    own imports -- accelerate, transformers, PIL -- are not installed);
  * the reference `IDDPM(..., return_startx=True)` around depth-2 reference models (fp32, CPU, seeded).

Sampler fixtures (`lcm_s*.pt`): the log_validation loop (train_pixart_lcm.py:124-133) for a batch of n with the toy denoiser
of oracle/dpm_oracle.py, every CPU draw recorded, the CPU generator state after the loop and the output.  Distillation
fixtures (`lcm_distill_*.pt`): one step of train_pixart_lcm.py:232-309 with DISTINCT seeded student / teacher / EMA weights,
pinning x_prev, target, both losses, gradient fingerprints (gen_golden_train.py format) for the Huber and the L2 loss and
fingerprints of the EMA after one `ema_update`; plus the reference's plan tensors (timesteps, scalings, solver tables).
Rerunning reproduces the files byte for byte.   python oracle/gen_golden_lcm.py
"""
import ast
import io
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dpm_oracle as do                   # noqa: E402
from oracle import pixart_oracle as po                # noqa: E402
from oracle.gen_golden import build_reference         # noqa: E402
from oracle.gen_golden_train import fingerprint_positions, train_inputs  # noqa: E402
from oracle.refshim import REFERENCE_ROOT, install_reference_shims  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SAMPLER_CASES = {"lcm_s4": dict(steps=4, n=2, hw=(8, 8)),          # log_validation's own call, batch 2
                 "lcm_s1": dict(steps=1, n=1, hw=(8, 8)),          # one step: no noise draw at all
                 "lcm_s2": dict(steps=2, n=1, hw=(8, 8)),
                 "lcm_s8": dict(steps=8, n=1, hw=(8, 8)),
                 "lcm_s4_nonsquare": dict(steps=4, n=1, hw=(8, 12))}
DISTILL_CASES = {"lcm_distill_d2": dict(cfg=dict(depth=2, input_size=32, pe_interpolation=0.5), batch=2, hw=(32, 32),
                                        lens=[300, 41], index=[0, 37])}
SEEDS = {"student": 0, "teacher": 1, "ema": 2}


def install_diffusers_stub() -> None:
    """The three diffusers symbols diffusion/lcm_scheduler.py imports, when diffusers itself is absent."""
    import importlib.util
    if "diffusers" in sys.modules or importlib.util.find_spec("diffusers") is not None:
        return
    import functools
    import inspect
    from collections import OrderedDict

    class ConfigMixin:
        pass

    class SchedulerMixin:
        pass

    class BaseOutput(OrderedDict):
        def __post_init__(self):
            for k, v in self.__dict__.items():
                self[k] = v

    def register_to_config(init):
        @functools.wraps(init)
        def wrapped(self, *args, **kwargs):
            bound = inspect.signature(init).bind(self, *args, **kwargs)
            bound.apply_defaults()
            self.config = types.SimpleNamespace(**{k: v for k, v in bound.arguments.items() if k != "self"})
            init(self, *args, **kwargs)
        return wrapped

    d = types.ModuleType("diffusers")
    d.ConfigMixin, d.SchedulerMixin = ConfigMixin, SchedulerMixin
    cu = types.ModuleType("diffusers.configuration_utils")
    cu.register_to_config = register_to_config
    ut = types.ModuleType("diffusers.utils")
    ut.BaseOutput = BaseOutput
    d.configuration_utils, d.utils = cu, ut
    sys.modules.update({"diffusers": d, "diffusers.configuration_utils": cu, "diffusers.utils": ut})


def training_script_defs() -> dict:
    """The top-level helper definitions of train_scripts/train_pixart_lcm.py, executed without the script's imports."""
    path = os.path.join(REFERENCE_ROOT, "train_scripts", "train_pixart_lcm.py")
    tree = ast.parse(open(path).read(), filename=path)
    wanted = {"DDIMSolver", "scalings_for_boundary_conditions", "extract_into_tensor", "append_dims", "ema_update"}
    body = [n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in wanted]
    assert {n.name for n in body} == wanted
    ns = {"torch": torch, "np": np, "nn": torch.nn}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns


def _save(obj, name):
    buf = io.BytesIO()
    torch.save(obj, buf)
    with open(os.path.join(OUT, name + ".pt"), "wb") as f:
        f.write(buf.getvalue())


def sampler_inputs(case, seed=0):
    g = torch.Generator().manual_seed(seed)
    n, (h, w) = case["n"], case["hw"]
    return torch.randn(n, 4, h, w, generator=g), torch.randn(n, 1, 6, 8, generator=g) * 0.5


def gen_sampler():
    from diffusion.lcm_scheduler import LCMScheduler
    for name, case in SAMPLER_CASES.items():
        x_T, cond = sampler_inputs(case)
        scheduler = LCMScheduler(beta_start=0.0001, beta_end=0.02, beta_schedule="linear", prediction_type="epsilon")
        scheduler.set_timesteps(case["steps"], 50)
        draws, randn = [], torch.randn

        def recording_randn(*a, **k):
            r = randn(*a, **k)
            draws.append(r.clone())
            return r
        torch.manual_seed(2000 + case["steps"])
        torch.randn = recording_randn
        try:
            latents, denoised = x_T.clone(), None
            for i, t in enumerate(scheduler.timesteps):                     # train_pixart_lcm.py:124-131
                ts = torch.full((case["n"],), t, dtype=torch.long)
                model_pred = do.toy_model(latents, ts, cond)[:, :4]
                latents, denoised = scheduler.step(model_pred, i, t, latents, return_dict=False)
        finally:
            torch.randn = randn
        _save(dict(case=case, seed=2000 + case["steps"], x_T=x_T, cond=cond, timesteps=scheduler.timesteps.clone(),
                   alphas_cumprod=scheduler.alphas_cumprod.clone(),
                   draws=torch.stack(draws) if draws else torch.zeros(0), rng_after=torch.get_rng_state(), out=denoised,
                   generator="oracle/gen_golden_lcm.py"), name)
        print(name, "timesteps", scheduler.timesteps.tolist(), "draws", len(draws))


def fingerprints(params):
    out = {}
    for n, v in params:
        flat = v.detach().flatten().float()
        out[n] = {"norm": flat.norm().clone(), "vals": flat[fingerprint_positions(flat.numel())].clone()}
    return out


def gen_distill():
    from diffusion import IDDPM
    ns = training_script_defs()
    diffusion = IDDPM(str(1000), learn_sigma=True, pred_sigma=True, snr=False, return_startx=True)
    solver = ns["DDIMSolver"](diffusion.alphas_cumprod, timesteps=1000, ddim_timesteps=50)
    scal, append_dims = ns["scalings_for_boundary_conditions"], ns["append_dims"]
    topk = 1000 // 50
    all_idx = torch.arange(50)
    all_start = solver.ddim_timesteps[all_idx]
    all_t = torch.where(all_start - topk < 0, torch.zeros_like(all_start), all_start - topk)
    plan = dict(ddim_timesteps=solver.ddim_timesteps.clone(), ddim_alpha_cumprods_prev=solver.ddim_alpha_cumprods_prev.clone(),
                scalings_start=torch.stack(scal(all_start)), scalings_t=torch.stack(scal(all_t)),
                sqrt_acp=ns["extract_into_tensor"](solver.ddim_alpha_cumprods_prev, all_idx, (50, 4, 1, 1)).sqrt().flatten(),
                sqrt_1macp=(1.0 - ns["extract_into_tensor"](solver.ddim_alpha_cumprods_prev, all_idx, (50, 4, 1, 1))).sqrt().flatten())
    for name, c in DISTILL_CASES.items():
        cfg = po.OracleConfig(**c["cfg"])
        models = {k: build_reference(cfg, po.synthetic_state_dict(cfg, seed=s)) for k, s in SEEDS.items()}
        student, teacher, ema = models["student"].train(), models["teacher"].eval(), models["ema"].eval()
        student.y_embedder.uncond_prob = 0.0          # token_drop is random and calls .cuda() (PixArt_blocks.py:394)
        for m in (teacher, ema):
            m.requires_grad_(False)
        latents, _, y, mask, _ = train_inputs(cfg, c["batch"], tuple(c["hw"]), [0] * c["batch"], c["lens"])
        g = torch.Generator().manual_seed(91)
        noise = torch.randn(latents.shape, generator=g)
        index = torch.tensor(c["index"], dtype=torch.long)
        bsz = latents.shape[0]
        uncond = student.y_embedder.y_embedding.repeat(bsz, 1, 1, 1)                    # train_pixart_lcm.py:191
        y_mask = mask
        # train_pixart_lcm.py:238-298, unchanged but for the autocast contexts (CPU fp32 here)
        start_timesteps = solver.ddim_timesteps[index]
        timesteps = start_timesteps - topk
        timesteps = torch.where(timesteps < 0, torch.zeros_like(timesteps), timesteps)
        c_skip_start, c_out_start = scal(start_timesteps)
        c_skip_start, c_out_start = [append_dims(x, latents.ndim) for x in [c_skip_start, c_out_start]]
        c_skip, c_out = scal(timesteps)
        c_skip, c_out = [append_dims(x, latents.ndim) for x in [c_skip, c_out]]
        w = 4.5 * torch.ones((bsz,))
        w = w.reshape(bsz, 1, 1, 1).to(dtype=latents.dtype)
        eps_s, pred_x_0, noisy_model_input = diffusion.training_losses(
            student, latents, start_timesteps, model_kwargs=dict(y=y, mask=y_mask, data_info=None), noise=noise)
        model_pred = c_skip_start * noisy_model_input + c_out_start * pred_x_0
        with torch.no_grad():
            cond_teacher_output, cond_pred_x0, _ = diffusion.training_losses(
                teacher, latents, start_timesteps, model_kwargs=dict(y=y, mask=y_mask, data_info=None), noise=noise)
            uncond_teacher_output, uncond_pred_x0, _ = diffusion.training_losses(
                teacher, latents, start_timesteps, model_kwargs=dict(y=uncond, mask=y_mask, data_info=None), noise=noise)
            pred_x0 = cond_pred_x0 + w * (cond_pred_x0 - uncond_pred_x0)
            pred_noise = cond_teacher_output + w * (cond_teacher_output - uncond_teacher_output)
            x_prev = solver.ddim_step(pred_x0, pred_noise, index)
        with torch.no_grad():
            eps_e, pred_x_0_e, _ = diffusion.training_losses(
                ema, x_prev.float(), timesteps, model_kwargs=dict(y=y, mask=y_mask, data_info=None), skip_noise=True)
            target = c_skip * x_prev + c_out * pred_x_0_e
        loss_l2 = torch.nn.functional.mse_loss(model_pred.float(), target.float(), reduction="mean")
        loss_huber = torch.mean(torch.sqrt((model_pred.float() - target.float()) ** 2 + 0.001 ** 2) - 0.001)
        loss_huber.backward(retain_graph=True)
        grads_huber = fingerprints((n, p.grad) for n, p in student.named_parameters())
        student.zero_grad(set_to_none=True)
        loss_l2.backward()
        grads_l2 = fingerprints((n, p.grad) for n, p in student.named_parameters())
        ns["ema_update"](ema, student, 0.95)
        _save(dict(case=name, cfg=c["cfg"], batch=c["batch"], hw=c["hw"], lens=c["lens"], seeds=SEEDS, index=index,
                   noise=noise, start=start_timesteps, t=timesteps, x_t=noisy_model_input.detach(),
                   eps_s=eps_s.detach().clone(), eps_c=cond_teacher_output.clone(), eps_u=uncond_teacher_output.clone(),
                   eps_e=eps_e.clone(), model_pred=model_pred.detach(), x_prev=x_prev, target=target, loss_huber=loss_huber.detach().clone(),
                   loss_l2=loss_l2.detach().clone(), grads_huber=grads_huber, grads_l2=grads_l2,
                   ema_after=fingerprints(ema.named_parameters()), plan=plan, generator="oracle/gen_golden_lcm.py"), name)
        print(name, "loss huber", float(loss_huber), "l2", float(loss_l2), "x_prev", x_prev.dtype, "target", target.dtype)


def main():
    install_reference_shims()
    install_diffusers_stub()
    os.makedirs(OUT, exist_ok=True)
    torch.use_deterministic_algorithms(True)
    torch.set_num_threads(1)
    gen_sampler()
    gen_distill()


if __name__ == "__main__":
    main()
