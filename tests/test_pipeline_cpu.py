"""Host side of `pixart_sigma_b200.pipeline` / `.generate`: prompt cleaning, the model constructor of inference.py, checkpoint
loaders, the uint8 conversion against torchvision, CLI parsing, and the CUDA-only checks."""
import json
import os

import pytest
import torch
from transformers import T5Tokenizer  # noqa: F401  (imported before the reference's timm stand-in, which its import probe rejects)

from oracle import pixart_oracle as po
from oracle.refshim import install_reference_shims, reference_available
from pixart_sigma_b200 import convert, generate, lib, pipeline
from pixart_sigma_b200.t5 import T5EncoderModel
from pixart_sigma_b200.vae import AutoencoderKL

TRICKY = ["a cat --ar 16:9", "a dog --hw 512:768 and more", "  spaces around  --aspect_ratio 1:2 --ar 3:4",
          "an --artistic painting", "no flags at all ", "--ar 1:1", "hyphen-ated --hw", "x --aspect_ratio 2:1--ar 1:2"]


def u8_formula(y: torch.Tensor) -> torch.Tensor:
    """pxa_vae_out_u8's conversion restated in fp32 torch ops."""
    v = y.float().clamp(-1, 1)
    v = (v + 1) / 2
    v = (v * 255 + 0.5).clamp(0, 255)
    return v.to(torch.uint8)


@pytest.mark.skipif(not reference_available(), reason="reference checkout not present")
def test_clean_prompt_matches_reference_prepare_prompt_ar():
    install_reference_shims()
    from diffusion.model.utils import prepare_prompt_ar
    ratios = {"0.5": [1448.0, 724.0], "1.0": [1024.0, 1024.0], "2.0": [724.0, 1448.0]}
    for p in TRICKY:
        assert pipeline.clean_prompt(p) == prepare_prompt_ar(p, ratios, show=False)[0].strip(), p


def test_clean_prompt_cases():
    assert pipeline.clean_prompt("a cat --ar 16:9") == "a cat"
    assert pipeline.clean_prompt("an --artistic painting") == "an"          # the script splits at any "--ar"
    assert pipeline.clean_prompt("  plain  ") == "plain"
    assert list(pipeline.get_chunks(list(range(5)), 2)) == [[0, 1], [2, 3], [4]]


@pytest.mark.parametrize("version", ["alpha", "sigma"])
@pytest.mark.parametrize("size", [256, 512, 1024, 2048])
def test_transformer_constructor_follows_inference_py(version, size):
    spec = pipeline.transformer_config(version, size)
    ms = size in (512, 1024, 2048) or version == "sigma"
    assert spec["name"] == ("PixArtMS_XL_2" if ms else "PixArt_XL_2")
    kw = spec["kwargs"]
    assert kw["input_size"] == size // 8 and kw["pe_interpolation"] == size / 512
    assert kw["model_max_length"] == {"alpha": 120, "sigma": 300}[version]
    assert kw.get("micro_condition", False) == (version == "alpha" and size == 1024)
    with pytest.raises(ValueError):
        pipeline.transformer_config("beta", size)


def _small_sd(micro=False):
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5, micro_condition=micro, model_max_length=300)
    return po.synthetic_state_dict(cfg, seed=1)


def test_pth_and_diffusers_checkpoints_load_key_for_key(tmp_path):
    sd = _small_sd()
    path = tmp_path / "ckpt.pth"
    torch.save({"state_dict": dict(sd)}, path)
    m, missing, unexpected = pipeline.load_transformer(str(path), "sigma", 256, device="cpu", depth=2)
    assert missing == ["pos_embed"] and unexpected == []
    assert m.dtype == torch.bfloat16 and not m.training
    got = m.state_dict()
    for k, v in sd.items():
        if k != "pos_embed":
            assert torch.equal(got[k], v.to(torch.bfloat16)), k
    from safetensors.torch import save_file
    (tmp_path / "hf" / "transformer").mkdir(parents=True)
    dsd = {k: v.contiguous() for k, v in convert.to_diffusers(sd).items()}
    save_file(dsd, str(tmp_path / "hf" / "transformer" / "diffusion_pytorch_model.safetensors"))
    m2, missing2, unexpected2 = pipeline.load_transformer(str(tmp_path / "hf"), "sigma", 256, device="cpu", depth=2)
    assert unexpected2 == [] and sorted(missing2) == ["pos_embed", "y_embedder.y_embedding"]
    got2 = m2.state_dict()
    for k in convert.from_diffusers(dsd):
        assert torch.equal(got2[k], got[k]), k
    torch.save(dict(sd), tmp_path / "bare.pth")
    with pytest.raises(ValueError):
        pipeline.load_transformer(str(tmp_path / "bare.pth"), "sigma", 256, device="cpu", depth=2)


def _write_sharded(folder, stem, sd, n_shards):
    from safetensors.torch import save_file
    os.makedirs(folder, exist_ok=True)
    keys = sorted(sd)
    weight_map = {}
    for i in range(n_shards):
        name = f"{stem}-{i + 1:05d}-of-{n_shards:05d}.safetensors"
        part = {k: sd[k].contiguous() for k in keys[i::n_shards]}
        save_file(part, os.path.join(folder, name))
        weight_map.update({k: name for k in part})
    with open(os.path.join(folder, f"{stem}.safetensors.index.json"), "w") as f:
        json.dump({"metadata": {}, "weight_map": weight_map}, f)


def test_sharded_t5_and_vae_load_in_bf16(tmp_path):
    from oracle.gen_golden_pipeline import VAE_CFG, synthetic_vae_state_dict, write_tokenizer
    from oracle.gen_golden_t5 import synthetic_t5_state_dict
    t5_cfg = dict(vocab_size=256, d_model=128, d_kv=32, d_ff=256, num_layers=2, num_heads=4)
    sd = synthetic_t5_state_dict(t5_cfg, seed=3)
    sd.pop("encoder.embed_tokens.weight")                           # tied to shared.weight: files may leave it out
    root = tmp_path / "pipe"
    _write_sharded(str(root / "text_encoder"), "model", sd, 3)
    with open(root / "text_encoder" / "config.json", "w") as f:
        json.dump(dict(t5_cfg, model_type="t5", feed_forward_proj="gated-gelu"), f)
    write_tokenizer(str(root))
    tok, enc = pipeline.load_text_encoder(str(root), device="cpu")
    assert isinstance(enc, T5EncoderModel) and enc.cfg["d_model"] == 128 and enc.cfg["num_layers"] == 2
    got = enc.state_dict()
    for k, v in sd.items():
        assert got[k].dtype == torch.bfloat16 and torch.equal(got[k], v.to(torch.bfloat16)), k
    assert enc.encoder.embed_tokens is enc.shared
    assert tok("a cat", return_tensors="pt").input_ids.shape[0] == 1

    vsd = synthetic_vae_state_dict(2)
    _write_sharded(str(root / "vae"), "diffusion_pytorch_model", vsd, 2)
    with open(root / "vae" / "config.json", "w") as f:
        json.dump(dict(VAE_CFG, block_out_channels=list(VAE_CFG["block_out_channels"]), scaling_factor=0.18215), f)
    vae = pipeline.load_vae(str(root / "vae"), device="cpu")
    assert isinstance(vae, AutoencoderKL) and vae.config.scaling_factor == 0.18215
    assert tuple(vae.config.block_out_channels) == VAE_CFG["block_out_channels"]
    gv = vae.state_dict()
    assert sorted(gv) == sorted(vsd)
    assert all(gv[k].dtype == torch.bfloat16 and torch.equal(gv[k], v.to(torch.bfloat16)) for k, v in vsd.items())
    vsd.pop("decoder.conv_out.bias")
    _write_sharded(str(tmp_path / "bad"), "diffusion_pytorch_model", vsd, 1)
    with open(tmp_path / "bad" / "config.json", "w") as f:
        json.dump(dict(VAE_CFG, block_out_channels=list(VAE_CFG["block_out_channels"])), f)
    with pytest.raises(RuntimeError, match="decoder.conv_out.bias"):
        pipeline.load_vae(str(tmp_path / "bad"), device="cpu")


def test_u8_formula_matches_torchvision_save_image_bytes(tmp_path):
    from PIL import Image
    from torchvision.utils import save_image
    g = torch.Generator().manual_seed(0)
    y = torch.randn(3, 37, 53, generator=g) * 0.8
    edges = torch.tensor([-1.5, -1.0, -0.999, -1 + 1 / 255, -0.5, 0.0, 1 / 510, 0.5, 0.999, 1.0, 1.5, 2.0 / 255 - 1])
    ks = torch.arange(256, dtype=torch.float32)
    y.view(-1)[:edges.numel()] = edges
    y.view(-1)[100:356] = (ks - 0.5) / 255 * 2 - 1                  # values that land on the rounding boundaries
    y.view(-1)[400:656] = ks / 255 * 2 - 1
    path = tmp_path / "img.png"                                      # lossless: the bytes save_image hands to PIL
    save_image(y, str(path), nrow=1, normalize=True, value_range=(-1, 1))
    want = torch.from_numpy(__import__("numpy").array(Image.open(path)))
    assert torch.equal(u8_formula(y.permute(1, 2, 0)), want)


def test_cli_parses_inference_py_arguments(tmp_path):
    a = generate.get_parser().parse_args([])
    assert (a.image_size, a.version, a.bs, a.cfg_scale, a.sampling_algo, a.seed, a.step, a.sdvae, a.cuda_graph) == \
        (1024, "sigma", 1, 4.5, "dpm-solver", 0, -1, False, False)
    a = generate.get_parser().parse_args(["--txt_file", "p.txt", "--image_size", "512", "--version", "alpha", "--model_path", "m.pth",
                                          "--pipeline_load_from", "pl", "--bs", "4", "--cfg_scale", "7", "--sampling_algo", "iddpm",
                                          "--seed", "9", "--step", "50", "--sdvae", "--height", "768", "--width", "1024",
                                          "--out_dir", "o", "--cuda_graph"])
    assert (a.txt_file, a.image_size, a.version, a.model_path, a.pipeline_load_from, a.bs, a.cfg_scale, a.sampling_algo, a.seed,
            a.step, a.sdvae, a.height, a.width, a.out_dir, a.cuda_graph) == \
        ("p.txt", 512, "alpha", "m.pth", "pl", 4, 7.0, "iddpm", 9, 50, True, 768, 1024, "o", True)
    with pytest.raises(SystemExit):
        generate.get_parser().parse_args(["--sampling_algo", "ddim"])
    (tmp_path / "p.txt").write_text("a cat --ar 1:1\nsecond line\n")
    assert generate.read_prompts(str(tmp_path / "p.txt")) == ["a cat --ar 1:1", "second line"]


def test_cpu_tensors_raise():
    m = pipeline.build_transformer("sigma", 256, device="cpu", depth=1)
    with pytest.raises(RuntimeError, match="CUDA"):
        pipeline.PixArtPipeline(m, None, None, None, "sigma", 256)
    x = torch.zeros(1, 4, 4, 128, dtype=torch.bfloat16)
    with pytest.raises(lib.PxaError):
        lib.vae_out_u8(x, torch.zeros(3, 3, 3, 128, dtype=torch.bfloat16), torch.zeros(3), torch.empty(1, 4, 4, 3, dtype=torch.uint8))
    from oracle.gen_golden_pipeline import VAE_CFG
    vae = AutoencoderKL(VAE_CFG).to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="sm_90a"):
        vae.decode_to_uint8(torch.zeros(1, 4, 4, 4))
