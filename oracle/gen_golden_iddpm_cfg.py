"""TEST INFRASTRUCTURE ONLY -- the classifier-free-guidance fixture of `pixart_sigma_b200.iddpm`, from the UNMODIFIED reference:
`IDDPM("10").p_sample_loop(model.forward_with_cfg, z.shape, z, clip_denoised=False, model_kwargs=dict(y=cat([caption, null_y]),
cfg_scale=4.5, data_info=..., mask=emb_masks))` as scripts/inference.py:89-101 calls it, around a depth-2 reference PixArtMS at
256px (latent 32 x 32) with n = 2 prompts and ragged caption masks, on CPU in fp32.  Weights and captions are the seeded
synthetic ones of oracle/pixart_oracle.py rounded to bf16, so the sm_90a model is built from exactly the same values; the
null caption is the model's own `y_embedder.y_embedding` (inference.py:84).  The final layer's variance rows are scaled by
`var_scale` so the learned variance stays in [-1, 1].  The sample still grows over the loop (rms 1 -> ~290): a model with
random weights is no denoiser, its eps is uncorrelated with the noise in x, so each step multiplies x by about
post_c1 * sqrt_recip_ac + post_c2 = 1 / sqrt(alpha_t), 1 / sqrt(alphas_cumprod[999]) ~ 157 over the loop, whatever the
weights' scale.  The comparison is relative, so the scale does not weaken it.

Stored: the case, the final sample `out` (all 2n rows), the first step's sample `x1` (the model input of the second call),
the timestep map and the timesteps the model was called with.  The latents, captions and per-step draws are regenerated from
the stored seeds by the tests: `torch.manual_seed(draw_seed)` then one `randn(2n, 4, 32, 32)` per step is the loop's stream.
Kept apart from oracle/gen_golden_iddpm.py so that rerunning one never rewrites the other's fixtures.
Needs the reference checkout (PIXART_REFERENCE_ROOT):   python oracle/gen_golden_iddpm_cfg.py"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pixart_oracle as po            # noqa: E402
from oracle.gen_golden import build_reference     # noqa: E402
from oracle.refshim import install_reference_shims  # noqa: E402

NAME = "iddpm_cfg_d2_s10"
CASE = dict(steps="10", n=2, hw=(32, 32), lens=[120, 37], cfg=4.5, clip=False, depth=2, input_size=32, pe_interpolation=0.5,
            weight_seed=0, var_scale=0.2, input_seed=7, z_seed=21, draw_seed=31)


def case_inputs(case=CASE):
    """(oracle config, bf16-rounded state dict, z (2n, 4, h, w), model_kwargs) of the fixture, on CPU."""
    cfg = po.OracleConfig(depth=case["depth"], input_size=case["input_size"], pe_interpolation=case["pe_interpolation"])
    sd = po.synthetic_state_dict(cfg, seed=case["weight_seed"])
    # the final layer's variance rows (output channel = row % 8 >= 4 after unpatchify) scaled so that the variance output
    # stays inside the learned range [-1, 1], where LEARNED_RANGE interpolates instead of extrapolating
    var = ((torch.arange(sd["final_layer.linear.weight"].shape[0]) % 8) >= 4).float()
    row_scale = 1 + (case["var_scale"] - 1) * var
    sd["final_layer.linear.weight"] = sd["final_layer.linear.weight"] * row_scale[:, None]
    sd["final_layer.linear.bias"] = sd["final_layer.linear.bias"] * row_scale
    sd = {k: v.to(torch.bfloat16).float() for k, v in sd.items()}
    n = case["n"]
    _, _, y, mask = po.synthetic_inputs(cfg, n, case["hw"], seed=case["input_seed"], lens=case["lens"])
    y = y.to(torch.bfloat16).float()
    null_y = sd["y_embedder.y_embedding"][None].repeat(n, 1, 1)[:, None]                 # inference.py:84
    z = torch.randn(n, 4, *case["hw"], generator=torch.Generator().manual_seed(case["z_seed"])).repeat(2, 1, 1, 1)
    hw = torch.tensor([[8.0 * case["hw"][0], 8.0 * case["hw"][1]]]).repeat(n, 1)
    kwargs = dict(y=torch.cat([y, null_y]), cfg_scale=case["cfg"], data_info={"img_hw": hw, "aspect_ratio": torch.ones(n, 1)},
                  mask=mask)
    return cfg, sd, z, kwargs


def main():
    install_reference_shims()
    from diffusion import IDDPM
    cfg, sd, z, kwargs = case_inputs()
    ref = build_reference(cfg, sd)
    xs, ts = [], []

    def model(x, timestep, **kw):
        xs.append(x.clone())
        ts.append(timestep.clone())
        return ref.forward_with_cfg(x, timestep, **kw)

    torch.manual_seed(CASE["draw_seed"])
    d = IDDPM(CASE["steps"])
    with torch.no_grad():
        out = d.p_sample_loop(model, z.shape, z, clip_denoised=CASE["clip"], model_kwargs=kwargs, progress=False, device="cpu")
    torch.save({"case": CASE, "out": out, "x1": xs[1], "timestep_map": list(d.timestep_map), "calls": torch.stack(ts),
                "generator": "oracle/gen_golden_iddpm_cfg.py", "reference_commit": "1ce521af"},
               os.path.join(ROOT, "tests", "golden", NAME + ".pt"))
    print(NAME, d.num_timesteps, "steps, |out| =", float(out.norm()), "|x1 - z| =", float((xs[1] - z).norm()))


if __name__ == "__main__":
    main()
