"""TEST INFRASTRUCTURE ONLY -- generate tests/golden/dmd_*.pt by running the UNMODIFIED reference DMD code from the reference
checkout that oracle/refshim.py locates:

  * `scripts/DMD/transformer_train/generate.py` (`generate_sample_1step`, `eps_to_mu`, `forward_model`) imported as is, with
    a stand-in `accelerate.utils.other.extract_model_from_parallel` (the identity: no wrapper here);
  * the statements of one step of `train_scripts/train_pixart_dmd.py` -- the one-step generator (:488-491), the
    distribution-matching loss (:493-571) and the fake model's denoising loss (:627-669) -- taken from the script's AST and
    executed in a namespace with `args` at the launcher's settings (scripts/run_pixart_dmd.py: cfg 3, start_ts 999,
    one_step_maxt 999, no regression, snr_gamma None, noise_offset 0), `F`, and a `DDPMScheduler` stand-in.  `init_noise` is
    drawn first by :484-485's own call, `torch.randn((b, 4, h, w))`, at the case's latent size: the script hard-codes 64 x 64
    (512 px), and 32 x 32 keeps the fixtures small;
  * depth-2 reference `PixArtMS` models (fp32, CPU, seeded) behind a thin adapter that gives them the diffusers
    `Transformer2DModel` call surface the script uses (`.config.sample_size` / `.config.out_channels`, `.sample`).
RESTATED, not from the reference tree (diffusers is not part of it): the `DDPMScheduler` stand-in (float32 linear-beta
`alphas_cumprod` and `add_noise`) and `EMAModel.step` (decay 0 on the first update, then min((1 + s) / (10 + s), 0.9999);
`s -= (1 - decay) (s - p)`).

Step fixtures (`dmd_step_*.pt`): the timesteps and fingerprints of the noise draws (from the CPU generator, in the script's
order; the seed regenerates them), latents, noisy latents, the eps channels of the real and fake outputs, weight, a coeff
fingerprint, both losses, gradient fingerprints (gen_golden_train.py format) of the generator (dm_loss) and of the fake
model (sg_loss), and the EMA after two updates (initialised from the EMA seed's weights, updated with the generator's and
then with the fake model's weights).  Sampling fixtures (`dmd_sample_*.pt`): `generate_sample_1step` at t = 400 (the app's
one-step sampler) and t = 999, with the toy denoiser of oracle/dpm_oracle.py and with a depth-2 model.
Rerunning reproduces the files byte for byte.   python oracle/gen_golden_dmd.py
"""
import ast
import io
import os
import sys
import types

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dpm_oracle as do                   # noqa: E402
from oracle import pixart_oracle as po                # noqa: E402
from oracle.gen_golden import build_reference         # noqa: E402
from oracle.gen_golden_lcm import fingerprints        # noqa: E402
from oracle.refshim import REFERENCE_ROOT, install_reference_shims  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
CFG = dict(depth=2, input_size=32, pe_interpolation=0.5, model_max_length=120)   # 32 x 32 latents, 120 caption tokens
# rng 1423 draws the DM timesteps [4, 997]: both ends of [1, 999)
STEP_CASES = {"dmd_step_d2": dict(seeds=dict(generator=0, real=1, fake=2, ema=3), lens=[120, 37], rng=1423),
              "dmd_step_d2_same": dict(seeds=dict(generator=0, real=0, fake=0, ema=3), lens=[120, 37], rng=1423)}
SAMPLE_CASES = {"dmd_sample_toy_t400": dict(model="toy", t=400, n=2, hw=(8, 8)),
                "dmd_sample_toy_t999": dict(model="toy", t=999, n=2, hw=(8, 8)),
                "dmd_sample_d2_t400": dict(model="d2", t=400, n=2, hw=(32, 32)),
                "dmd_sample_d2_t999": dict(model="d2", t=999, n=2, hw=(32, 32))}
ARGS = dict(use_dm=True, use_regression=False, noise_offset=0, start_ts=999, one_step_maxt=999, fix_noise_ts=None,
            prediction_type=None, cfg=3.0, snr_gamma=None)


class DDPMSchedulerStandIn:
    """RESTATED from diffusers' DDPMScheduler (not in the reference tree): float32 linear betas, `add_noise`."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02):
        self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)

    def add_noise(self, original_samples, noise, timesteps):
        alphas_cumprod = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)
        timesteps = timesteps.to(original_samples.device)
        sqrt_alpha_prod = (alphas_cumprod[timesteps] ** 0.5).flatten()
        while len(sqrt_alpha_prod.shape) < len(original_samples.shape):
            sqrt_alpha_prod = sqrt_alpha_prod.unsqueeze(-1)
        sqrt_one_minus_alpha_prod = ((1 - alphas_cumprod[timesteps]) ** 0.5).flatten()
        while len(sqrt_one_minus_alpha_prod.shape) < len(original_samples.shape):
            sqrt_one_minus_alpha_prod = sqrt_one_minus_alpha_prod.unsqueeze(-1)
        return sqrt_alpha_prod * original_samples + sqrt_one_minus_alpha_prod * noise


class DiffusersSurface(torch.nn.Module):
    """A reference PixArtMS (or the toy denoiser) called as the script calls a diffusers Transformer2DModel."""

    def __init__(self, net, sample_size, out_channels):
        super().__init__()
        self.net = net
        self.config = types.SimpleNamespace(sample_size=sample_size, out_channels=out_channels)

    def forward(self, hidden_states, timestep=None, encoder_hidden_states=None, encoder_attention_mask=None,
                added_cond_kwargs=None):
        di = None
        if added_cond_kwargs and added_cond_kwargs.get("resolution") is not None:
            di = dict(img_hw=added_cond_kwargs["resolution"], aspect_ratio=added_cond_kwargs["aspect_ratio"])
        out = self.net(hidden_states, timestep, encoder_hidden_states[:, None], mask=encoder_attention_mask, data_info=di)
        return types.SimpleNamespace(sample=out)


def import_generate():
    acc, utils, other = (types.ModuleType(n) for n in ("accelerate", "accelerate.utils", "accelerate.utils.other"))
    other.extract_model_from_parallel = lambda model: model
    acc.utils, utils.other = utils, other
    sys.modules.update({"accelerate": acc, "accelerate.utils": utils, "accelerate.utils.other": other})
    import importlib.util
    path = os.path.join(REFERENCE_ROOT, "scripts", "DMD", "transformer_train", "generate.py")
    spec = importlib.util.spec_from_file_location("dmd_generate", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def step_statements():
    """The training loop's statements at train_pixart_dmd.py:488-571 and :627-669, as one compiled module."""
    path = os.path.join(REFERENCE_ROOT, "train_scripts", "train_pixart_dmd.py")
    src = open(path).read()
    tree = ast.parse(src, filename=path)
    loop = next(n for n in ast.walk(tree) if isinstance(n, ast.For) and "train_dataloader" in ast.unparse(n.iter))
    body = next(n for n in loop.body if isinstance(n, ast.With)).body
    picked = [n for n in body if 488 <= n.lineno <= 571 or 627 <= n.lineno <= 669]
    heads = [ast.unparse(n).split("\n")[0] for n in picked]
    assert heads[0].startswith("latents = generate_sample_1step"), heads
    assert "if args.use_dm:" in heads and heads[-1] == "if args.snr_gamma is None:", heads
    assert any(h.startswith("latents_for_fake = latents.detach()") for h in heads), heads
    return compile(ast.Module(body=picked, type_ignores=[]), path, "exec")


def _save(obj, name):
    buf = io.BytesIO()
    torch.save(obj, buf)
    with open(os.path.join(OUT, name + ".pt"), "wb") as f:
        f.write(buf.getvalue())


def step_inputs(cfg, b, lens, seed=0):
    _, _, y, mask = po.synthetic_inputs(cfg, b, (cfg.input_size, cfg.input_size), seed=seed, lens=lens)
    g = torch.Generator().manual_seed(seed + 5)
    uncond_y = torch.randn(1, cfg.model_max_length, 4096, generator=g)
    uncond_mask = torch.zeros(1, cfg.model_max_length)
    uncond_mask[0, 0] = 1.0                                   # the empty prompt: one (eos) token
    return y.squeeze(1), mask.float(), uncond_y, uncond_mask


def gen_step(gen_mod, code):
    cfg = po.OracleConfig(**CFG)
    for name, c in STEP_CASES.items():
        sds = {k: po.synthetic_state_dict(cfg, seed=s) for k, s in c["seeds"].items()}
        nets = {k: build_reference(cfg, sds[k]) for k in ("generator", "real", "fake")}
        model, model_real, model_fake = (DiffusersSurface(nets[k], cfg.input_size, cfg.out_channels)
                                         for k in ("generator", "real", "fake"))
        for m in (model, model_fake):
            m.train()
            m.net.y_embedder.uncond_prob = 0.0                # the diffusers transformer drops no captions
        model_real.eval().requires_grad_(False)
        y, y_mask, uncond_y, uncond_mask = step_inputs(cfg, 2, c["lens"])
        ns = dict(torch=torch, F=F, args=types.SimpleNamespace(**ARGS), accelerator=types.SimpleNamespace(device="cpu"),
                  batch={}, weight_dtype=torch.float32, y=y, y_mask=y_mask, model=model, model_real=model_real,
                  model_fake=model_fake, noise_scheduler=DDPMSchedulerStandIn(),
                  generate_sample_1step=gen_mod.generate_sample_1step, forward_model=gen_mod.forward_model,
                  negative_prompt_embeds=uncond_y, negative_prompt_attention_masks=uncond_mask)
        torch.manual_seed(c["rng"])
        h = w = cfg.input_size
        ns["init_noise"] = torch.randn((y.shape[0], 4, h, w), dtype=torch.float32, device="cpu")   # :484-485
        exec(code, ns)
        ns["dm_loss"].backward()
        ns["sgloss"].backward()
        grads_gen = fingerprints((n, p.grad) for n, p in nets["generator"].named_parameters())
        grads_fake = fingerprints((n, p.grad) for n, p in nets["fake"].named_parameters())
        # EMAModel.step (RESTATED): shadow from the EMA seed; update 1 (decay 0) with the generator, update 2 with the fake
        shadow = {k: v.clone() for k, v in sds["ema"].items()}
        decays = []
        for k, src in enumerate((sds["generator"], sds["fake"])):
            s = max(0, k + 1 - 1)
            decay = 0.0 if s <= 0 else min((1 + s) / (10 + s), 0.9999)
            decays.append(decay)
            for n, v in shadow.items():
                v.sub_((1 - decay) * (v - src[n]))
        _save(dict(case=name, cfg=CFG, seeds=c["seeds"], lens=c["lens"], rng=c["rng"], args=ARGS,
                   draws=fingerprints((k, ns[k]) for k in ("init_noise", "noise", "noise_for_fake")), t=ns["timesteps"],
                   t_f=ns["timesteps_for_fake"], rng_after=torch.get_rng_state(),
                   latents=ns["latents"].detach().clone(), noisy=ns["noisy_latents"].detach().clone(),
                   real_out=ns["model_real_output"][:, :4].clone(), fake_out=ns["model_fake_output"][:, :4].clone(),
                   weight=ns["weight"].reshape(-1).clone(), coeff=fingerprints([("coeff", ns["coeff"])])["coeff"], dm_loss=ns["dm_loss"].detach().clone(),
                   sg_loss=ns["sgloss"].detach().clone(), grads_gen=grads_gen, grads_fake=grads_fake, ema_decays=decays,
                   ema_after=fingerprints(shadow.items()), generator="oracle/gen_golden_dmd.py"), name)
        print(name, "t", ns["timesteps"].tolist(), "t_f", ns["timesteps_for_fake"].tolist(), "dm_loss", float(ns["dm_loss"].detach()),
              "sg_loss", float(ns["sgloss"].detach()), "weight", ns["weight"].flatten().tolist())


def gen_sample(gen_mod):
    sched = DDPMSchedulerStandIn()
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    for name, c in SAMPLE_CASES.items():
        g = torch.Generator().manual_seed(c["t"])
        n, (h, w) = c["n"], c["hw"]
        x_T = torch.randn(n, 4, h, w, generator=g)
        if c["model"] == "toy":
            cond = torch.randn(n, 6, 8, generator=g) * 0.5
            net = lambda x, t, y, mask=None, data_info=None: do.toy_model(x, t, y)
            model, y, mask = DiffusersSurface(net, 0, 4), cond, None
        else:
            _, _, y, mask = po.synthetic_inputs(cfg, n, (h, w), lens=[300, 77])
            y = y.squeeze(1)
            model = DiffusersSurface(build_reference(cfg, po.synthetic_state_dict(cfg, seed=0)), cfg.input_size, 8)
        with torch.no_grad():
            out = gen_mod.generate_sample_1step(model, sched, x_T, c["t"], y, mask)
        _save(dict(case=c, x_T=x_T, cond=y if c["model"] == "toy" else None, alphas_cumprod=sched.alphas_cumprod.clone(), out=out,
                   generator="oracle/gen_golden_dmd.py"), name)
        print(name, "out abs mean", float(out.abs().mean()))


def main():
    install_reference_shims()
    os.makedirs(OUT, exist_ok=True)
    torch.use_deterministic_algorithms(True)
    torch.set_num_threads(1)
    gen_mod = import_generate()
    gen_sample(gen_mod)
    gen_step(gen_mod, step_statements())


if __name__ == "__main__":
    main()
