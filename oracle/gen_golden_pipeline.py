"""TEST INFRASTRUCTURE ONLY -- end-to-end fixtures of `pixart_sigma_b200.pipeline` from the UNMODIFIED reference
scripts/inference.py, run with `runpy` and its own command line on CPU in fp32, one fixture per sampler:

    inference.py --image_size 256 --version sigma --bs 2 --cfg_scale 4.5 --seed 3 --sampling_algo {dpm-solver,sa-solver,iddpm}
                 --step {5,-,10} --txt_file prompts.txt --model_path .../ckpt.pth --pipeline_load_from .../pipeline

Only the loaders are stand-ins, all seeded, and none of them changes what the script computes:
  * `find_model` loads a real `{'state_dict': ...}` checkpoint written here: `po.synthetic_state_dict` of a depth-2 model,
    with `y_embedder.y_proj.fc1` and `y_embedding` re-drawn for the tiny T5's width and the final layer's variance rows
    scaled so that the learned variance stays in [-1, 1] (as oracle/gen_golden_iddpm_cfg.py does); values rounded to bf16;
  * `diffusion.model.nets.PixArtMS_XL_2` builds the reference's PixArtMS at depth 2 with caption_channels = the T5 width;
  * `transformers.T5EncoderModel.from_pretrained` gives transformers' own T5 encoder with `synthetic_t5_state_dict` weights;
  * `T5Tokenizer.from_pretrained` is transformers' tokenizer on a SentencePiece model trained here (`write_tokenizer`);
  * `diffusers.models.AutoencoderKL.from_pretrained` decodes with oracle/vae_oracle.py on `synthetic_vae_state_dict`;
  * the model's and the VAE's `.to(torch.float16)` are ignored, so everything runs in fp32 (the script's
    `samples.to(weight_dtype)` still rounds the latents to fp16 before the VAE, as it does on a GPU);
  * `SASolverSampler.register_buffer` keeps `alphas_cumprod` on the CPU (sa_sampler.py:24-28 moves it to CUDA);
  * `diffusers.utils.torch_utils.randn_tensor` and `mmcv.build_from_cfg`, imported by the dataset package, are never called.
`save_image` is captured (its image argument), and so is the initial latent draw of `torch.randn`.  Stored per fixture: the
case, the cleaned prompts, z, the CPU generator's state right after z, the VAE input, every 8th row and column of the
images (`images_sub`; the test decodes the stored VAE input again with oracle/vae_oracle.py for the full images, and checks
them against these samples) and the weights' seeds (the test rebuilds the weights).  z cannot be redrawn from the seed on the CPU, since building the models draws from the same
generator after `set_env`; the per-step draws of the stochastic samplers are the stream from the stored state on.
Rerunning reproduces the files byte for byte.   Needs the reference checkout:   python oracle/gen_golden_pipeline.py"""
import io
import os
import runpy
import sys
import tempfile
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pixart_oracle as po             # noqa: E402
from oracle import vae_oracle                       # noqa: E402
from oracle.gen_golden_t5 import synthetic_t5_state_dict  # noqa: E402

PROMPTS = ["a small red fox sleeping in the snow under a pine tree, soft light --ar 16:9",
           "neon city --hw 512:768"]
T5_CFG = dict(vocab_size=256, d_model=256, d_kv=64, d_ff=512, num_layers=2, num_heads=4)
VAE_CFG = dict(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=(64, 64, 128, 128), layers_per_block=2,
               norm_num_groups=32, scaling_factor=0.13025)
COMMON = dict(image_size=256, version="sigma", bs=2, cfg_scale=4.5, seed=3, depth=2, weight_seed=0, t5_seed=11, vae_seed=5,
              var_scale=0.2)
CASES = {"pipeline_dpm": dict(COMMON, sampling_algo="dpm-solver", step=5),
         "pipeline_sa": dict(COMMON, sampling_algo="sa-solver", step=-1),
         "pipeline_iddpm": dict(COMMON, sampling_algo="iddpm", step=10)}
TOKENIZER_TEXT = ["a photo of a cat sitting on a red chair", "an astronaut riding a horse on the moon, digital art",
                  "close-up portrait of an old man with a beard", "a watercolor painting of a lighthouse at sunset",
                  "a small red fox sleeping in the snow under a pine tree", "neon city street at night in the rain"]


def write_tokenizer(folder: str) -> str:
    """A SentencePiece unigram model trained on TOKENIZER_TEXT (deterministic), as `{folder}/tokenizer/spiece.model`."""
    import sentencepiece as spm
    buf = io.BytesIO()
    spm.SentencePieceTrainer.train(sentence_iterator=iter(TOKENIZER_TEXT * 20), model_writer=buf, vocab_size=120,
                                   model_type="unigram", pad_id=0, eos_id=1, unk_id=2, bos_id=-1, num_threads=1, minloglevel=2,
                                   hard_vocab_limit=False)
    os.makedirs(os.path.join(folder, "tokenizer"), exist_ok=True)
    path = os.path.join(folder, "tokenizer", "spiece.model")
    with open(path, "wb") as f:
        f.write(buf.getvalue())
    return path


def transformer_state_dict(case: dict) -> dict:
    """The depth-2 PixArtMS weights of the fixture (bf16-rounded fp32), caption_channels = T5_CFG['d_model']."""
    S = case["image_size"]
    cfg = po.OracleConfig(depth=case["depth"], input_size=S // 8, pe_interpolation=S / 512)
    sd = po.synthetic_state_dict(cfg, seed=case["weight_seed"])
    g = torch.Generator().manual_seed(case["weight_seed"] + 1000)
    D = T5_CFG["d_model"]
    sd["y_embedder.y_proj.fc1.weight"] = torch.randn(cfg.hidden_size, D, generator=g) * D ** -0.5
    sd["y_embedder.y_embedding"] = torch.randn(cfg.model_max_length, D, generator=g) * D ** -0.5
    var = ((torch.arange(sd["final_layer.linear.weight"].shape[0]) % 8) >= 4).float()
    row_scale = 1 + (case["var_scale"] - 1) * var
    sd["final_layer.linear.weight"] = sd["final_layer.linear.weight"] * row_scale[:, None]
    sd["final_layer.linear.bias"] = sd["final_layer.linear.bias"] * row_scale
    return {k: v.to(torch.bfloat16).float() for k, v in sd.items()}


def synthetic_vae_state_dict(seed: int, cfg: dict = VAE_CFG) -> dict:
    """Seeded VAE weights in diffusers' AutoencoderKL layout for `cfg` (bf16-rounded fp32): matrices ~ N(0, 1 / fan_in),
    norm weights 1 + 0.1 N(0, 1), biases 0.1 N(0, 1); keys in sorted order."""
    from pixart_sigma_b200.vae import AutoencoderKL
    with torch.device("meta"):
        shapes = {k: tuple(v.shape) for k, v in AutoencoderKL(cfg).state_dict().items()}
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k in sorted(shapes):
        shp = shapes[k]
        if len(shp) > 1:
            v = torch.randn(shp, generator=g) * (torch.Size(shp[1:]).numel() ** -0.5)
        elif "norm" in k and k.endswith("weight"):
            v = 1 + 0.1 * torch.randn(shp, generator=g)
        else:
            v = 0.1 * torch.randn(shp, generator=g)
        sd[k] = v.to(torch.bfloat16).float()
    return sd


class _Fp32:
    """`.to(...)` keeps fp32 and CPU (the script casts the model and the VAE to fp16)."""

    def to(self, *args, **kwargs):
        return self


def _install_loader_shims(case: dict, captured: dict):
    import transformers                                    # before the timm stand-in, which transformers' probe rejects
    from transformers import T5EncoderModel, T5Tokenizer    # noqa: F401
    from oracle.refshim import install_reference_shims
    install_reference_shims()
    sys.modules["mmcv"].build_from_cfg = lambda *a, **k: None

    class _VaeShim(_Fp32):
        def __init__(self):
            self.sd = synthetic_vae_state_dict(case["vae_seed"])
            self.config = types.SimpleNamespace(scaling_factor=VAE_CFG["scaling_factor"])

        @classmethod
        def from_pretrained(cls, *a, **k):
            return cls()

        def decode(self, z):
            captured["vae_in"] = z.clone()
            return types.SimpleNamespace(sample=vae_oracle.decode(self.sd, z.float()))

    diffusers = types.ModuleType("diffusers")
    models = types.ModuleType("diffusers.models")
    models.AutoencoderKL = _VaeShim
    utils = types.ModuleType("diffusers.utils")
    tu = types.ModuleType("diffusers.utils.torch_utils")
    tu.randn_tensor = lambda *a, **k: None
    diffusers.models, diffusers.utils, utils.torch_utils = models, utils, tu
    sys.modules.update({"diffusers": diffusers, "diffusers.models": models, "diffusers.utils": utils,
                        "diffusers.utils.torch_utils": tu})

    transformers = sys.modules["transformers"]             # the lazy module replaces itself there on import
    real_t5 = getattr(transformers.T5EncoderModel, "real", transformers.T5EncoderModel)

    class _T5Shim:
        real = real_t5

        @staticmethod
        def from_pretrained(*a, **k):
            hf = real_t5(transformers.T5Config(feed_forward_proj="gated-gelu", dropout_rate=0.0, **T5_CFG)).eval()
            missing, unexpected = hf.load_state_dict(synthetic_t5_state_dict(T5_CFG, case["t5_seed"]), strict=False)
            assert not missing and not unexpected, (missing, unexpected)
            return hf
    transformers.T5EncoderModel = _T5Shim

    import diffusion.model.nets as nets
    from diffusion.model.nets.PixArtMS import PixArtMS

    def depth2(**kwargs):
        m = PixArtMS(depth=case["depth"], hidden_size=1152, patch_size=2, num_heads=16, caption_channels=T5_CFG["d_model"], **kwargs)
        m.to = types.MethodType(_Fp32.to, m)
        return m
    nets.PixArtMS_XL_2 = depth2
    from diffusion import SASolverSampler
    SASolverSampler.register_buffer = lambda self, name, attr: setattr(self, name, attr)   # the reference moves it to CUDA

    import torchvision.utils
    torchvision.utils.save_image = lambda t, path, **kw: captured["images"].append(t.clone())


def run_case(name: str, case: dict, work: str) -> dict:
    captured = dict(images=[], z=[])
    _install_loader_shims(case, captured)
    pipe = os.path.join(work, "pipeline")
    write_tokenizer(pipe)
    ckpt = os.path.join(work, "models", "ckpt", "ckpt.pth")
    os.makedirs(os.path.dirname(ckpt), exist_ok=True)
    torch.save({"state_dict": transformer_state_dict(case)}, ckpt)
    txt = os.path.join(work, "prompts.txt")
    with open(txt, "w") as f:
        f.write("\n".join(PROMPTS) + "\n")
    S = case["image_size"]
    randn = torch.randn

    def recording_randn(*size, **kw):      # the initial latents: default-generator latent draws but set_env's (1, 4, S, S)
        out = randn(*size, **kw)
        shape = tuple(size[0]) if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)) else tuple(size)
        if "generator" not in kw and len(shape) == 4 and shape[1] == 4 and shape != (1, 4, S, S):
            captured["z"].append(out.clone())
            captured["rng_after_z"] = torch.get_rng_state()
        return out
    torch.randn = recording_randn
    argv = ["inference.py", "--image_size", str(S), "--version", case["version"], "--bs", str(case["bs"]),
            "--cfg_scale", str(case["cfg_scale"]), "--seed", str(case["seed"]), "--sampling_algo", case["sampling_algo"],
            "--step", str(case["step"]), "--txt_file", txt, "--model_path", ckpt, "--pipeline_load_from", pipe]
    old_argv, old_cwd = sys.argv, os.getcwd()
    sys.argv = argv
    os.chdir(work)
    try:
        runpy.run_path(os.path.join(po_reference_root(), "scripts", "inference.py"), run_name="__main__")
    finally:
        sys.argv = old_argv
        os.chdir(old_cwd)
        torch.randn = randn
    assert len(captured["z"]) == 1, [tuple(z.shape) for z in captured["z"]]
    return {"case": case, "prompts": PROMPTS, "clean_prompts": [p.split("--ar")[0].split("--hw")[0].strip() for p in PROMPTS],
            "t5_cfg": T5_CFG, "vae_cfg": VAE_CFG, "z": captured["z"][0], "rng_after_z": captured["rng_after_z"], "vae_in": captured["vae_in"],
            "images_sub": torch.stack(captured["images"])[..., ::8, ::8].clone(), "generator": "oracle/gen_golden_pipeline.py", "reference_commit": "1ce521af"}


def po_reference_root() -> str:
    from oracle.refshim import REFERENCE_ROOT
    return REFERENCE_ROOT


def main():
    torch.set_num_threads(1)
    for name, case in CASES.items():
        with tempfile.TemporaryDirectory() as work:
            fix = run_case(name, case, work)
        torch.save(fix, os.path.join(ROOT, "tests", "golden", name + ".pt"))
        torch.set_grad_enabled(True)                      # set_env turned it off
        print(name, "z", tuple(fix["z"].shape), "images_sub", tuple(fix["images_sub"].shape), "|vae_in| =", float(fix["vae_in"].float().norm()))


if __name__ == "__main__":
    main()
