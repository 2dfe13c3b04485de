"""GPU tests (-m gpu) of the native IDDPM loop: the fused step kernel (pxa_iddpm_step) against a float64 restatement of the
torch loop's formula, the loop against the reference fixtures (tests/golden/iddpm_sample_*.pt from oracle/gen_golden_iddpm.py
with its toy denoiser, tests/golden/iddpm_cfg_d2_s10.pt from oracle/gen_golden_iddpm_cfg.py with a depth-2 PixArtMS and
classifier-free guidance), the random stream, CUDA-graph capture and the absence of host syncs.

Tolerances: step kernel vs float64 1e-6 (fp32 arithmetic with FMA contraction); toy loop vs fixture 1e-5 (up to 100 steps of
the above); same-seed native vs torch loop 1e-6; loop around the sm_90a PixArtMS: see that test."""
import os
import sys
import zlib

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.gen_golden_iddpm import CASES, toy_model           # noqa: E402
from oracle.gen_golden_iddpm_cfg import NAME as CFG_NAME       # noqa: E402
from oracle.gen_golden_iddpm_cfg import case_inputs            # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"

if torch.cuda.is_available():
    from pixart_sigma_b200 import PixArtMS, lib
    from pixart_sigma_b200.iddpm import IDDPM, _STEP_KEYS


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def _gold(name):
    return torch.load(os.path.join(GOLD, name + ".pt"))


def _step64(out, img, noise, guided, clip, cfg, st):
    """float64 restatement of forward_with_cfg's mix + p_mean_variance + p_sample (iddpm.py), scalars as the kernel gets them."""
    o, x = out.double().cpu(), img.double().cpu()
    N = x.shape[0]
    eps, v = o[:, :4].clone(), o[:, 4:]
    if guided:
        n = N // 2
        ec, eu = eps[:n, :3], eps[n:, :3]
        mixed = eu + cfg * (ec - eu)
        eps[:n, :3], eps[n:, :3] = mixed, mixed
    frac = (v + 1) / 2
    logvar = frac * st["log_beta"] + (1 - frac) * st["post_logvar"]
    x0 = st["sqrt_recip_ac"] * x - st["sqrt_recipm1_ac"] * eps
    if clip:
        x0 = x0.clamp(-1, 1)
    mean = st["post_c1"] * x0 + st["post_c2"] * x
    new = mean + (torch.exp(0.5 * logvar) * noise.double().cpu() if noise is not None else 0)
    return new, (torch.cat([new[:N // 2], new[:N // 2]]) if guided else None)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("guided", [True, False])
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("step", ["first", "middle", "t0"])
def test_step_kernel_matches_float64_formula(dtype, guided, clip, step):
    g = torch.Generator().manual_seed(zlib.crc32(f"{dtype}{guided}{clip}{step}".encode()))
    n = int(torch.randint(1, 4, (1,), generator=g))
    h, w = (int(v) for v in torch.randint(5, 40, (2,), generator=g))
    if (h * w) % 256 == 0:
        w += 1
    N = 2 * n if guided else n
    st = IDDPM("100").plan()[{"first": 0, "middle": 50, "t0": 99}[step]]
    assert (st["t"] == 0) == (step == "t0")
    full = torch.randn(N, 10, h, w, generator=g)                     # a channel slice: (N, 8, h, w), batch stride 10 hw
    full[:, 4:] = full[:, 4:].tanh()                                 # variance channels in the learned range
    out = full.to(dtype).to(DEV)[:, :8]
    img, noise = (torch.randn(N, 4, h, w, generator=g).to(DEV) for _ in range(2))
    noise = None if step == "t0" else noise
    nxt = torch.full_like(img, float("nan")) if guided else None
    want, want_in = _step64(out, img, noise, guided, clip, 4.5, st)
    got = lib.iddpm_step(out, img.clone(), noise, nxt, guided=guided, clip=clip, cfg_scale=4.5,
                         **{k: st[k] for k in _STEP_KEYS})
    assert _rel(got, want) < 1e-6
    if guided:
        assert _rel(nxt, want_in) < 1e-6
        assert torch.equal(nxt[:n], nxt[n:]) and torch.equal(nxt[:n], got[:n])


def test_step_kernel_rejects_bad_arguments():
    z = torch.zeros(2, 8, 4, 4, device=DEV)
    img = torch.zeros(2, 4, 4, 4, device=DEV)
    args = lib.IddpmStepArgs(model_out=z.data_ptr(), img=img.data_ptr(), noise=None, next_in=None, out_batch_stride=128, n=1,
                             hw=16, out_dtype=lib.DTYPE_F32, guided=1, clip=0)
    assert lib.load().pxa_iddpm_step(lib.C.byref(args), lib._stream()) == -1       # guided needs next_in; nothing launched
    args.guided, args.out_dtype = 0, 7
    assert lib.load().pxa_iddpm_step(lib.C.byref(args), lib._stream()) == -1       # unknown dtype


def _toy_draws(fix):
    """The per-step draws of the fixture's seeded reference run, regenerated on the CPU (one randn_like(img) per step)."""
    torch.manual_seed(100 + fix["seed"])
    return [torch.randn(fix["z"].shape) for _ in fix["timestep_map"]]


@pytest.mark.parametrize("name", sorted(CASES))
def test_loop_with_toy_denoiser_matches_reference_fixture(name):
    fix = _gold(name)
    d = IDDPM(fix["steps"])
    draws = _toy_draws(fix)
    calls = []
    kw = dict(clip_denoised=fix["clip"], model_kwargs=dict(scale=0.9), device=DEV, noise_draws=draws)
    out = d.p_sample_loop(toy_model(calls), fix["z"].shape, fix["z"].to(DEV), **kw)
    assert out.is_cuda and out.dtype == torch.float32
    assert torch.equal(torch.stack(calls).cpu(), fix["calls"])               # original timestep indices, int64
    err = _rel(out, fix["out"])
    assert err < 1e-5, f"{name}: rel_err vs reference fixture = {err:.3e}"
    graphed = d.p_sample_loop(toy_model(), fix["z"].shape, fix["z"].to(DEV), cuda_graph=True, **kw)
    assert torch.equal(graphed, out)


def test_same_seed_native_and_torch_loops_draw_the_same_numbers():
    """x_T and every step's randn_like(img) come from the default CUDA generator in the reference's order."""
    d = IDDPM("25")
    shape = (3, 4, 9, 7)
    torch.cuda.manual_seed(17)
    native = d.p_sample_loop(toy_model(), shape, None, clip_denoised=False, model_kwargs=dict(scale=0.9), device=DEV)
    torch.cuda.manual_seed(17)
    *_, last = d.p_sample_loop_progressive(toy_model(), shape, None, clip_denoised=False, model_kwargs=dict(scale=0.9),
                                           device=DEV)
    err = _rel(native, last["sample"])
    assert err < 1e-6, f"native vs torch loop, same seed: rel_err = {err:.3e}"


def test_graphed_equals_eager_for_a_seed_and_replays_draw_fresh_noise():
    d = IDDPM("20")
    shape = (2, 4, 8, 8)
    kw = dict(clip_denoised=True, model_kwargs=dict(scale=0.9), device=DEV)
    model = toy_model()                                          # one callable: the captured loop is keyed on it
    torch.cuda.manual_seed(7)
    eager = d.p_sample_loop(model, shape, None, **kw)
    torch.cuda.manual_seed(7)
    graphed = d.p_sample_loop(model, shape, None, cuda_graph=True, **kw)
    assert torch.equal(graphed, eager) and d.last_capture_s is not None
    torch.cuda.manual_seed(7)
    replay = d.p_sample_loop(model, shape, None, cuda_graph=True, **kw)
    assert torch.equal(replay, eager) and len(d._graphs) == 1
    fresh = d.p_sample_loop(model, shape, None, cuda_graph=True, **kw)
    assert _rel(fresh, eager) > 1e-2


def test_loop_runs_without_autograd_whatever_the_grad_mode():
    """As the reference loop (gaussian_diffusion.py:493 runs under th.no_grad()): with grad mode on and a model whose
    parameters require grad, the denoiser must still see grad mode off, or PixArtMS.forward would take its training path."""
    base, w, seen = toy_model(), torch.ones((), device=DEV, requires_grad=True), []

    def model(x, timestep, **kw):
        seen.append(torch.is_grad_enabled())
        return base(x, timestep, **kw) * w
    d = IDDPM("10")
    z = torch.randn(2, 4, 8, 8, device=DEV)
    with torch.enable_grad():
        eager = d.p_sample_loop(model, z.shape, z, clip_denoised=False, model_kwargs=dict(scale=0.9), device=DEV)
        graphed = d.p_sample_loop(model, z.shape, z, clip_denoised=False, model_kwargs=dict(scale=0.9), device=DEV,
                                  cuda_graph=True)
    assert seen and not any(seen)
    assert not eager.requires_grad and not graphed.requires_grad


def test_eager_loop_adds_no_host_sync():
    d = IDDPM("10")
    z = torch.randn(2, 4, 8, 8, device=DEV)
    kw = dict(clip_denoised=False, model_kwargs=dict(scale=0.9), device=DEV)
    d.p_sample_loop(toy_model(), z.shape, z, **kw)                 # plan, timestep upload
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        d.p_sample_loop(toy_model(), z.shape, z, **kw)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_cfg_loop_around_the_sm90_model_matches_reference_fixture():
    """scripts/inference.py's call -- `IDDPM("10").p_sample_loop(model.forward_with_cfg, z.shape, z, clip_denoised=False,
    model_kwargs=dict(y=cat([caption, null_y]), cfg_scale=4.5, data_info=..., mask=...))` -- on a depth-2 sm_90a PixArtMS at
    256px with n = 2 and ragged masks, vs the unmodified reference loop around the fp32 reference model on the same
    bf16-rounded weights (tests/golden/iddpm_cfg_d2_s10.pt), with the fixture's draws replayed.

    Bound.  The native loop differs from the fixture only through the bf16 forward (the step is fp32 on both sides).  One
    step with the sm_90a forward, started from the fixture's x_T with its first draw, gives the first-step error s1 against
    the reference's first sample.  A step's coefficient on its input sample, post_c1 * sqrt_recip_ac + post_c2 =
    1 / sqrt(alpha_t), scales the sample and an error carried in it alike, so a relative error made at one step is carried
    forward at about its size, and each of the S = 10 steps adds one of about s1: the bound is 2 * S * s1, the factor 2 for
    the model's response to its perturbed input.  The same loop with fp16 model outputs (the script's `weight_dtype`) is
    held to the same bound.  Against the torch loop around the same sm_90a model (fp32 outputs) with the same seeded draws:
    both loops start from the same forward, so their first samples differ only in fp32 rounding (the kernel contracts into
    FMAs; 1e-6).  From the second step on, those last-bit differences flip bf16 roundings inside the forward, so each later
    step adds at most one bf16-forward error: the whole loop is held to (S - 1) * s1, under half the fixture bound."""
    fix = _gold(CFG_NAME)
    case = fix["case"]
    n, S = case["n"], len(fix["timestep_map"])
    cfg, sd, z, kw = case_inputs(case)
    with torch.device(DEV):
        m = PixArtMS(depth=case["depth"], input_size=case["input_size"], pe_interpolation=case["pe_interpolation"],
                     model_max_length=cfg.model_max_length)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and missing == ["pos_embed"]
    m = m.to(torch.bfloat16).eval()
    kw = dict(kw, y=kw["y"].to(DEV), mask=kw["mask"].to(DEV), data_info={k: v.to(DEV) for k, v in kw["data_info"].items()})
    torch.manual_seed(case["draw_seed"])
    draws = [torch.randn(z.shape) for _ in range(S)]
    zc = z.to(DEV)
    d = IDDPM(case["steps"])

    st = d.plan()[0]
    with torch.no_grad():
        out0 = m.forward(torch.cat([zc[:n], zc[:n]]), d._timesteps(zc.device, 2 * n)[0], kw["y"], kw["mask"],
                         data_info=kw["data_info"])
    x1 = lib.iddpm_step(out0, zc.clone(), draws[0].to(DEV), torch.empty_like(zc), guided=True, clip=False,
                        cfg_scale=case["cfg"], **{k: st[k] for k in _STEP_KEYS})
    s1 = _rel(x1, fix["x1"])
    bound = 2 * S * s1

    call = dict(clip_denoised=case["clip"], model_kwargs=kw, device=DEV)
    launches = lib.launch_count()
    out = d.p_sample_loop(m.forward_with_cfg, z.shape, zc, noise_draws=draws, **call)
    assert lib.launch_count() - launches >= S * (2 * 11 + 1)          # S x (2 blocks x 11 kernels + the step kernel)
    err = _rel(out, fix["out"])
    msg = f"IDDPM 10-step CFG loop, depth-2 model at 256px: first-step error {s1:.3e}, bound {bound:.3e}"
    assert err < bound, f"{msg}, rel_err vs reference = {err:.3e}"
    graphed = d.p_sample_loop(m.forward_with_cfg, z.shape, zc, noise_draws=draws, cuda_graph=True, **call)
    assert _rel(graphed, out) < 1e-5

    m.output_dtype = torch.float32
    torch.cuda.manual_seed(3)
    native = d.p_sample_loop(m.forward_with_cfg, z.shape, zc, **call)
    torch.cuda.manual_seed(3)
    glue = [o["sample"] for o in d.p_sample_loop_progressive(m.forward_with_cfg, z.shape, zc, **call)]
    torch.cuda.manual_seed(3)
    first_draw = torch.randn(z.shape, device=DEV)
    with torch.no_grad():
        out0 = m.forward(torch.cat([zc[:n], zc[:n]]), d._timesteps(zc.device, 2 * n)[0], kw["y"], kw["mask"],
                         data_info=kw["data_info"])
    x1_native = lib.iddpm_step(out0, zc.clone(), first_draw, torch.empty_like(zc), guided=True, clip=False,
                               cfg_scale=case["cfg"], **{k: st[k] for k in _STEP_KEYS})
    err_first = _rel(x1_native, glue[0])
    assert err_first < 1e-6, f"{msg}, first step vs the torch loop on the same model = {err_first:.3e}"
    err_glue = _rel(native, glue[-1])
    assert err_glue < (S - 1) * s1, f"{msg}, rel_err vs the torch loop on the same model = {err_glue:.3e}"

    m.output_dtype = torch.float16
    out16 = d.p_sample_loop(m.forward_with_cfg, z.shape, zc, noise_draws=draws, **call)
    err16 = _rel(out16, fix["out"])
    assert err16 < bound, f"{msg}, fp16 outputs: rel_err vs reference = {err16:.3e}"
    graphs = len(d._graphs)                                          # the output dtype is part of the captured loop's key
    graphed16 = d.p_sample_loop(m.forward_with_cfg, z.shape, zc, noise_draws=draws, cuda_graph=True, **call)
    assert len(d._graphs) == graphs + 1 and _rel(graphed16, out16) < 1e-5
    print(f"{msg}; rel_err bf16 out {err:.3e}, fp16 out {err16:.3e}, vs torch loop {err_glue:.3e} (first step {err_first:.3e})")
