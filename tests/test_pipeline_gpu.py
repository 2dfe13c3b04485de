"""`pxa_vae_out_u8` against float64, and the text-to-image pipeline end to end against the unmodified inference.py
(tests/golden/pipeline_*.pt, oracle/gen_golden_pipeline.py): images, random stream, host syncs, CUDA graphs, real sizes."""
import os

import pytest
import torch
import torch.nn.functional as F
from transformers import T5Tokenizer  # noqa: F401  (imported before the reference's timm stand-in, which its import probe rejects)

from oracle.gen_golden_pipeline import (CASES, PROMPTS, T5_CFG, VAE_CFG, synthetic_vae_state_dict, transformer_state_dict,
                                        write_tokenizer)
from oracle import vae_oracle
from oracle.gen_golden_t5 import synthetic_t5_state_dict
from pixart_sigma_b200 import generate, lib, pipeline
from pixart_sigma_b200.t5 import T5EncoderModel
from pixart_sigma_b200.vae import SDXL_VAE_CONFIG, AutoencoderKL

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def u8_formula(y: torch.Tensor) -> torch.Tensor:
    v = y.float().clamp(-1, 1)
    v = (v + 1) / 2
    v = (v * 255 + 0.5).clamp(0, 255)
    return v.to(torch.uint8)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("B,H,W,Cin,pad", [(1, 8, 32, 128, 0), (3, 13, 37, 128, 0), (1, 1, 1, 8, 0), (2, 33, 65, 64, 0),
                                           (2, 17, 23, 128, 8), (1, 9, 40, 24, 16), (1, 1024, 1024, 128, 0)])
def test_vae_out_u8_matches_float64(B, H, W, Cin, pad):
    """y within 1/2 ulp + n 2^-24 (|b| + sum |h w|), n = 9 Cin + 1 terms (fp32 FMA chain); u8 = the formula on the kernel's own y,
    bit for bit.  Input pixels padded with NaN channels (pad > 0) and an output buffer banded by sentinels check the addressing."""
    g = torch.Generator().manual_seed(B * 1000 + H + W + Cin)
    h = (torch.randn(B, H, W, Cin, generator=g) * 0.7).to(torch.bfloat16)
    w = (torch.randn(3, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).to(torch.bfloat16)
    b = torch.randn(3, generator=g) * 0.1
    store = torch.full((B, H, W, Cin + pad), float("nan"), dtype=torch.bfloat16, device=DEV)
    store[..., :Cin] = h.to(DEV)
    x = store[..., :Cin]
    band = 4096
    u8_store = torch.full((2 * band + B * H * W * 3,), 0xA5, dtype=torch.uint8, device=DEV)
    f_store = torch.full((2 * band + B * H * W * 3,), -7.0, device=DEV)
    u8 = u8_store[band:band + B * H * W * 3].view(B, H, W, 3)
    y = f_store[band:band + B * H * W * 3].view(B, H, W, 3)
    lib.vae_out_u8(x, w.permute(0, 2, 3, 1).contiguous().to(DEV), b.to(DEV), u8, y)
    torch.cuda.synchronize()
    assert bool((u8_store[:band] == 0xA5).all()) and bool((u8_store[-band:] == 0xA5).all())
    assert bool((f_store[:band] == -7.0).all()) and bool((f_store[-band:] == -7.0).all())
    hd, wd = h.to(DEV).double().permute(0, 3, 1, 2), w.to(DEV).double()
    want = F.conv2d(hd, wd, b.to(DEV).double(), padding=1).permute(0, 2, 3, 1)
    mag = F.conv2d(hd.abs(), wd.abs(), b.to(DEV).double().abs(), padding=1).permute(0, 2, 3, 1)
    ulp = torch.finfo(torch.float32).eps * want.abs().float().clamp_min(torch.finfo(torch.float32).tiny).double()
    bound = 0.5 * ulp + (9 * Cin + 1) * 2.0 ** -24 * mag
    err = (y.double() - want).abs()
    assert bool((err <= bound).all()), f"max err / bound = {float((err / bound).max()):.3f}"
    assert torch.equal(u8, u8_formula(y))


def test_vae_out_u8_rejects_bad_arguments():
    x = torch.zeros(1, 4, 4, 12, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(lib.PxaError, match="multiple of 8"):
        lib.vae_out_u8(x, torch.zeros(3, 3, 3, 12, dtype=torch.bfloat16, device=DEV), torch.zeros(3, device=DEV),
                       torch.empty(1, 4, 4, 3, dtype=torch.uint8, device=DEV))


# ------------------------------------------------------------------------------------------------- the pipeline
def _pipe(tmp_path, case, *, image_size=256, depth=2):
    write_tokenizer(str(tmp_path))
    tok = T5Tokenizer.from_pretrained(str(tmp_path), subfolder="tokenizer")
    m = pipeline.build_transformer("sigma", image_size, DEV, depth=depth, caption_channels=T5_CFG["d_model"])
    if depth == 2:
        missing, unexpected = m.load_state_dict(transformer_state_dict(case), strict=False)
        assert missing == ["pos_embed"] and not unexpected
    m = m.to(torch.bfloat16).eval()
    enc = T5EncoderModel(T5_CFG)
    enc.load_state_dict(synthetic_t5_state_dict(T5_CFG, case["t5_seed"]), strict=False)
    enc = enc.to(DEV, torch.bfloat16).eval()
    vae = AutoencoderKL(VAE_CFG)
    vae.load_state_dict(synthetic_vae_state_dict(case["vae_seed"]))
    vae = vae.to(DEV, torch.bfloat16).eval()
    return pipeline.PixArtPipeline(m, tok, enc, vae, "sigma", image_size)


def _replay(case, gold):
    """The script's z and, from the CPU generator's state after it, the sampler's per-step draws (randn_like)."""
    z = gold["z"]
    torch.set_rng_state(gold["rng_after_z"])
    if case["sampling_algo"] == "iddpm":
        return z, [[torch.randn_like(z.repeat(2, 1, 1, 1)) for _ in range(case["step"])]]
    if case["sampling_algo"] == "sa-solver":
        torch.randn_like(z)                                               # the sampler's discarded draw
        return z, [[torch.randn_like(z) for _ in range(pipeline.SA_SOLVER_STEPS)]]
    return z, None


def _script_images(case, gold):
    """The script's saved images: its fp16 VAE input decoded again by the fp32 oracle VAE it ran with, checked against the
    fixture's samples of every 8th row and column (1e-4: the CPU convolutions' summation order depends on the thread
    count and the instruction set; 4e-6 to 6e-6 between one thread and several)."""
    with torch.no_grad():
        images = vae_oracle.decode(synthetic_vae_state_dict(case["vae_seed"]), gold["vae_in"].float())
    assert _rel(images[..., ::8, ::8], gold["images_sub"]) < 1e-4
    return images


@pytest.mark.parametrize("name", sorted(CASES))
def test_pipeline_matches_unmodified_inference_script(name, tmp_path):
    """Latents and images against the script's, with its z and draws replayed.  Bounds: the sampler fixtures' 2e-2 normwise on
    the latents (the fixture's latents are the fp16 VAE input the script makes, times the scaling factor, 2^-11 from fp16),
    and on the VAE's fp32 output 3e-2 (the latent error plus the bf16 VAE's 6e-3 of tests/test_vae_gpu.py)."""
    gold = torch.load(os.path.join(GOLD, name + ".pt"))
    case = gold["case"]
    pipe = _pipe(tmp_path, case)
    z, draws = _replay(case, gold)
    res = pipe.generate(PROMPTS, sampling_algo=case["sampling_algo"], steps=case["step"], cfg_scale=case["cfg_scale"], seed=None,
                        bs=case["bs"], x_T=z, noise_draws=draws, return_float=True, return_latents=True)
    assert res["prompts"] == gold["clean_prompts"]
    assert res["images"].shape == (2, 256, 256, 3) and res["images"].dtype == torch.uint8 and res["images"].is_cuda
    lat_err = _rel(res["latents"].cpu(), gold["vae_in"].double() * VAE_CFG["scaling_factor"])
    images = _script_images(case, gold)
    img_err = _rel(res["float"].cpu(), images)
    u8_gold = u8_formula(images.permute(0, 2, 3, 1))
    mismatch = float((res["images"].cpu().int() - u8_gold.int()).abs().float().mean())
    print(f"{name}: latents rel_err {lat_err:.3e}, VAE output rel_err {img_err:.3e}, mean |u8 diff| {mismatch:.3f}")
    assert lat_err < 2e-2 and img_err < 3e-2
    assert torch.equal(res["images"], u8_formula(res["float"].permute(0, 2, 3, 1)))


def test_seeded_latents_are_the_device_stream_and_graphs_are_bitwise(tmp_path):
    """A seed's latents are `torch.manual_seed(s); torch.randn(...)` on the device, and `cuda_graph=True` samples the same
    latents bit for bit.  Two decodes of the same latents are not bitwise equal: the GroupNorm kernel sums its statistics with
    floating-point atomics, in no fixed order.  On the first H100 runs 0.7 % of the values moved, by one or two levels, with
    these fixtures' large random-weight latents; the pixels are held to a mean difference of 0.05 levels."""
    case = CASES["pipeline_dpm"]
    pipe = _pipe(tmp_path, case)
    call = dict(sampling_algo="dpm-solver", steps=3, bs=2, return_latents=True)
    seeded = pipe.generate(PROMPTS, seed=7, **call)
    torch.manual_seed(7)
    z = torch.randn(2, 4, 32, 32, device=DEV)
    injected = pipe.generate(PROMPTS, seed=None, x_T=z, **call)
    assert torch.equal(seeded["latents"], injected["latents"])
    for algo, steps in (("dpm-solver", 3), ("sa-solver", None), ("iddpm", 4)):
        if algo == "dpm-solver":
            draws = None
        elif algo == "sa-solver":
            draws = [[torch.randn(2, 4, 32, 32) for _ in range(pipeline.SA_SOLVER_STEPS)]]
        else:
            draws = [[torch.randn(4, 4, 32, 32) for _ in range(steps)]]
        kw = dict(sampling_algo=algo, steps=steps, bs=2, seed=None, x_T=z, noise_draws=draws, return_latents=True)
        eager = pipe.generate(PROMPTS, **kw)
        graphed = pipe.generate(PROMPTS, cuda_graph=True, **kw)
        assert torch.equal(eager["latents"], graphed["latents"]), algo
        diff = (eager["images"].int() - graphed["images"].int()).abs()
        assert int(diff.max()) <= 8 and float(diff.float().mean()) < 5e-2, algo


@pytest.mark.parametrize("algo", ["dpm-solver", "sa-solver", "iddpm"])
def test_no_host_sync_between_token_upload_and_final_copy(algo, tmp_path):
    pipe = _pipe(tmp_path, CASES["pipeline_dpm"])
    call = dict(sampling_algo=algo, steps=3 if algo != "sa-solver" else None, bs=1, seed=1)
    pipe.generate(PROMPTS[:1], **call)                          # first use: tokenizer, allocator and kernel set-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = pipe.generate(PROMPTS, **call)["images"]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert out.cpu().shape == (2, 256, 256, 3)


def test_xl2_generates_1024px_jpegs_through_the_cli(tmp_path):
    """An XL/2-sized model (28 blocks, width 1152; random weights) at 1024 px with the SDXL-VAE geometry, through the CLI."""
    from PIL import Image
    case = CASES["pipeline_dpm"]
    pipe = _pipe(tmp_path, case, image_size=1024, depth=28)
    vae = AutoencoderKL(SDXL_VAE_CONFIG)
    vae.load_state_dict(synthetic_vae_state_dict(1, SDXL_VAE_CONFIG))
    pipe.vae = vae.to(DEV, torch.bfloat16).eval()
    txt = tmp_path / "prompts.txt"
    txt.write_text("a lighthouse at dusk --ar 1:1\nan astronaut riding a horse\n")
    paths = generate.main(["--txt_file", str(txt), "--image_size", "1024", "--bs", "2", "--step", "2", "--seed", "3",
                           "--out_dir", str(tmp_path / "out")], pipeline=pipe)
    assert [os.path.basename(p) for p in paths] == ["a lighthouse at dusk.jpg", "an astronaut riding a horse.jpg"]
    for p in paths:
        with Image.open(p) as im:
            assert im.format == "JPEG" and im.size == (1024, 1024) and im.mode == "RGB"
