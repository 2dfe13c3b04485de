"""GPU tests (-m gpu) of the SA-Solver sampler: the fused step kernel (pxa_sa_solver_step) and the sampling loop of
pixart_sigma_b200/sa_sampler.py against the oracle restatement (oracle/sa_oracle.py) and the reference fixtures
(tests/golden/sa_*.pt, written by oracle/gen_golden_sa.py from the unmodified reference).

Tolerances: step kernel vs the fp32 formula 1e-6 (fp32 arithmetic, reciprocal instead of division, FMA contraction); loop with
the deterministic toy denoiser vs the reference fixture 1e-5 (up to 25 evaluations of the above); loop around the sm_90a
PixArtMS vs the oracle loop around the oracle forward: see that test."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dpm_oracle as do            # noqa: E402
from oracle import pixart_oracle as po         # noqa: E402
from oracle import sa_oracle as so             # noqa: E402
from oracle.gen_golden_sa import CASES         # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"

if torch.cuda.is_available():
    from pixart_sigma_b200 import PixArtMS, lib
    from pixart_sigma_b200.sa_sampler import SASolverSampler


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm())


def _gold(name):
    return torch.load(os.path.join(GOLD, name + ".pt"))


def _call(g, **kw):
    """The sampler arguments of a fixture, on the device (built once per test: a captured loop is keyed on the addresses of
    the conditioning tensors)."""
    case = g["case"]
    args = dict(S=case["steps"], batch_size=case["n"], shape=(4,) + case["hw"], eta=case["eta"], conditioning=g["cond"].to(DEV),
                unconditional_conditioning=g["uncond"].to(DEV), unconditional_guidance_scale=case["cfg"], model_kwargs={},
                x_T=g["x_T"].to(DEV), noise=[d.to(DEV) for d in g["draws"][1:]])
    args.update(kw)
    return args


def _sample(solver, args, **kw):
    out, extra = solver.sample(**dict(args, **kw))
    assert extra is None
    return out


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("guided", [True, False])
@pytest.mark.parametrize("form", ["first", "deterministic", "stochastic"])
def test_step_kernel_matches_formula(dtype, guided, form):
    g = torch.Generator().manual_seed(4)
    n, h, w = 3, 24, 20
    full = torch.randn((2 if guided else 1) * n, 8, h, w, generator=g).to(dtype).to(DEV)   # learn-sigma output
    out = full[:, :4]                                                                   # the view forward_with_dpmsolver returns
    x, xp, mp, nc, npn = (torch.randn(n, 4, h, w, generator=g).to(DEV) for _ in range(5))
    k = dict(cfg_scale=4.5, sigma=0.83, alpha=0.557, c_x=0.93, c_m0=0.31, c_m1=-0.12, c_noise=0.27, p_x=0.88, p_m0=0.35,
             p_m1=-0.09, p_noise=0.22)
    if form == "first":                     # i = 0: identity corrector, order-1 predictor; m_prev is garbage and must not be read
        k.update(c_x=1.0, c_m0=0.0, c_m1=0.0, c_noise=0.0, p_m1=0.0)
        mp = torch.full_like(mp, float("nan"))
    if form != "stochastic":
        k.update(c_noise=0.0, p_noise=0.0)
    if guided:
        eu, ec = out.float().chunk(2)
        eps = eu + k["cfg_scale"] * (ec - eu)
    else:
        eps = out.float()
    m = (xp - k["sigma"] * eps) / k["alpha"]
    mp_ = torch.nan_to_num(mp)
    xc = k["c_x"] * x + k["c_m0"] * m + k["c_m1"] * mp_ + k["c_noise"] * nc
    xn = k["p_x"] * xc + k["p_m0"] * m + k["p_m1"] * mp_ + k["p_noise"] * npn
    gx, gxp, gmp = x.clone(), xp.clone(), mp.clone()
    lib.sa_solver_step(out, gx, gxp, gmp, nc if k["c_noise"] else None, npn if k["p_noise"] else None, guided=guided, **k)
    assert _rel(gx, xc) < 1e-6
    assert _rel(gxp, xn) < 1e-6
    assert _rel(gmp, m) < 1e-6


def test_step_kernel_requires_noise_for_a_nonzero_coefficient():
    z = torch.zeros(1, 4, 8, 8, device=DEV)
    k = dict(guided=False, cfg_scale=1.0, sigma=0.5, alpha=0.8, c_x=1.0, c_m0=0.0, c_m1=0.0, c_noise=0.0, p_x=1.0, p_m0=0.1,
             p_m1=0.0, p_noise=0.3)
    args = lib.SaStepArgs(model_out=z.data_ptr(), x=z.data_ptr(), x_pred=z.data_ptr(), m_prev=z.data_ptr(), noise_c=None,
                          noise_p=None, out_batch_stride=256, n=1, hw=64, out_dtype=lib.DTYPE_F32, guided=0,
                          cfg_scale=1.0, sigma=0.5, inv_alpha=1.25, c_x=1.0, p_x=1.0, p_m0=0.1, p_noise=0.3)
    assert lib.load().pxa_sa_solver_step(lib.C.byref(args), lib._stream()) == -1      # PXA_ERR_ARG, nothing launched
    with pytest.raises(AssertionError):
        lib.sa_solver_step(z, z.clone(), z.clone(), z.clone(), None, None, **k)


@pytest.mark.parametrize("name", sorted(CASES))
def test_loop_with_toy_denoiser_matches_reference_fixture(name):
    g = _gold(name)
    solver = SASolverSampler(do.toy_model, device=DEV)
    args = _call(g)
    out = _sample(solver, args)
    assert out.shape == g["out"].shape and _rel(out, g["out"]) < 1e-5
    graphed = _sample(solver, args, cuda_graph=True)
    again = _sample(solver, args, cuda_graph=True)                 # replay of the cached graph
    assert len(solver._graphs) == 1
    assert torch.equal(graphed, again) and _rel(graphed, g["out"]) < 1e-5


def test_rng_stream_matches_the_reference_draw_order():
    """x_T = randn(size), one discarded randn_like, then one draw per step (diffusion/sa_sampler.py:70-71,
    diffusion/model/sa_solver.py:785,850): with the same seed, drawing inside the sampler equals replaying those draws."""
    g = _gold("sa_s7_eta05")
    case = g["case"]
    size = (case["n"], 4) + case["hw"]
    solver = SASolverSampler(do.toy_model, device=DEV)
    args = _call(g)
    torch.cuda.manual_seed(123)
    drawn = _sample(solver, args, x_T=None, noise=None)
    torch.cuda.manual_seed(123)
    draws = [torch.randn(size, device=DEV)] + [torch.randn(size, device=DEV) for _ in range(case["steps"] + 1)]
    replayed = _sample(solver, args, x_T=draws[0], noise=draws[2:])
    assert torch.equal(drawn, replayed)
    want = so.sample(do.toy_model, draws[0].cpu(), g["cond"], g["uncond"], case["cfg"], case["steps"], case["eta"],
                     [d.cpu() for d in draws[2:]])
    assert _rel(drawn, want) < 1e-5


def test_same_seed_eager_and_graphed_agree_and_replays_draw_fresh_noise():
    g = _gold("sa_s25_eta1")
    solver = SASolverSampler(do.toy_model, device=DEV)
    args = _call(g, x_T=None, noise=None)
    torch.cuda.manual_seed(7)
    eager = _sample(solver, args)
    torch.cuda.manual_seed(7)
    graphed = _sample(solver, args, cuda_graph=True)
    assert _rel(graphed, eager) < 1e-6
    torch.cuda.manual_seed(7)
    replay = _sample(solver, args, cuda_graph=True)              # cached graph, same seed: same draws
    assert _rel(replay, eager) < 1e-6 and len(solver._graphs) == 1
    fresh = _sample(solver, args, cuda_graph=True)               # generator advanced: different draws
    assert _rel(fresh, eager) > 1e-2


def test_eager_loop_adds_no_host_sync():
    g = _gold("sa_s5_eta0")
    solver = SASolverSampler(do.toy_model, device=DEV)
    args = _call(g, noise=None)
    _sample(solver, args)                                        # lazy initialisation, plan cache
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _sample(solver, args)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_unguided_sampling_is_one_conditional_evaluation_per_step():
    """No unconditional input (or guidance scale 1): one conditional evaluation per step (sa_solver.py:311-312); the fixture
    was sampled with guidance scale 1 by the reference."""
    g = _gold("sa_s6_cfg1")
    batches = []

    def spy(x, t, c, **kw):
        batches.append(x.shape[0])
        return do.toy_model(x, t, c, **kw)

    solver = SASolverSampler(spy, device=DEV)
    out = _sample(solver, _call(g, unconditional_conditioning=None, unconditional_guidance_scale=4.5))
    assert batches == [g["case"]["n"]] * g["case"]["steps"]
    assert _rel(out, g["out"]) < 1e-5
    want = so.sample(do.toy_model, g["x_T"], g["cond"], None, 4.5, g["case"]["steps"], g["case"]["eta"], list(g["draws"][1:]))
    assert _rel(out, want) < 1e-5


def test_loop_around_the_sm90_model_matches_oracle_loop():
    """6-step (eta 1, replayed noise) CFG sampling of a depth-2 PixArtMS at 256px (latent 32x32) on the sm_90a kernels, called
    as scripts/inference.py:123-133 calls the sampler, vs the oracle loop around the fp32 oracle forward on the same
    bf16-rounded weights.  Bound 2e-2, as for the DPM-Solver++ loop: 6 denoiser evaluations at the model's ~3e-3 each,
    amplified by the solver's 1/alpha factors; the stochastic steps add the same noise to both sides.  The first run on an
    H100 80GB HBM3 (700 W) measured 1.08e-2 (the 4-step DPM-Solver++ loop: 0.96e-2)."""
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    sd = {k: v.to(torch.bfloat16).float() for k, v in po.synthetic_state_dict(cfg, seed=0).items()}
    z, _, y, mask = po.synthetic_inputs(cfg, 1, (32, 32), seed=5, lens=[77])
    null_y = po.synthetic_inputs(cfg, 1, (32, 32), seed=6)[2]
    y, null_y = y.to(torch.bfloat16).float(), null_y.to(torch.bfloat16).float()
    S = 6
    gen = torch.Generator().manual_seed(11)
    noise = [torch.randn(z.shape, generator=gen) for _ in range(S)]
    with torch.device(DEV):
        m = PixArtMS(depth=2, input_size=32, pe_interpolation=0.5, model_max_length=300)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and missing == ["pos_embed"]
    m = m.to(torch.bfloat16).eval()
    kw = dict(data_info=None, mask=mask.to(DEV))
    solver = SASolverSampler(m.forward_with_dpmsolver, device=DEV)
    call = dict(S=S, batch_size=1, shape=(4, 32, 32), eta=1, conditioning=y.to(DEV), unconditional_conditioning=null_y.to(DEV),
                unconditional_guidance_scale=4.5, model_kwargs=kw, x_T=z.to(DEV), noise=[e.to(DEV) for e in noise])
    launches = lib.launch_count()
    out = solver.sample(**call)[0]
    assert lib.launch_count() - launches >= S * (2 * 11 + 1)          # S x (2 blocks x 11 kernels + the step kernel)

    def oracle_model(x, t, c, **kwargs):
        return po.forward_with_dpmsolver(sd, cfg, x, t, c, data_info=None, mask=mask)
    want = so.sample(oracle_model, z, y, null_y, 4.5, S, 1, noise)
    err = _rel(out, want)
    assert err < 2e-2, f"SA-Solver 6-step loop, depth-2 model at 256px: rel_err vs oracle loop = {err:.3e}"
    graphed = solver.sample(**call, cuda_graph=True)[0]
    assert _rel(graphed, out) < 1e-5
