"""CPU tests of the SA-Solver sampler: the oracle restatement (oracle/sa_oracle.py) against fixtures produced by the unmodified
reference `SASolverSampler` (oracle/gen_golden_sa.py), the product's host-side plan against the oracle's coefficients, the
step-argument struct against the header, argument rejection, and the reference install."""
import ctypes
import os
import subprocess
import sys
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dpm_oracle as do             # noqa: E402
from oracle import refshim                      # noqa: E402
from oracle import sa_oracle as so              # noqa: E402
from oracle.gen_golden_sa import CASES          # noqa: E402
from pixart_sigma_b200 import lib, sa_sampler   # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_fixture(name):
    """Same float32 operations in the same order as the reference: bit-level agreement is expected, 1e-6 leaves room for
    elementwise differences between torch builds."""
    g = torch.load(os.path.join(GOLD, name + ".pt"))
    case = g["case"]
    assert case == CASES[name]
    calls = []

    def spy(x, t, c, **kw):
        calls.append((float(t[0]), x.shape[0]))
        return do.toy_model(x, t, c, **kw)

    assert g["draws"].shape[0] == case["steps"] + 1                  # one discarded draw at init + one per step
    out, x1 = so.sample(spy, g["x_T"], g["cond"], g["uncond"], case["cfg"], case["steps"], case["eta"], list(g["draws"][1:]),
                        return_first_corrected=True)
    assert len(calls) == case["steps"]                                # one denoiser evaluation per step, none at t_S
    assert torch.allclose(torch.tensor([t for t, _ in calls]), g["model_times"], atol=1e-3)
    rows = case["n"] * (1 if case["cfg"] == 1.0 else 2)              # unguided: the conditional rows alone
    assert all(b == rows for _, b in calls)
    assert _rel(out, g["out"]) < 1e-6
    assert _rel(x1, g["x_1"]) < 1e-6


def test_model_times_and_stochastic_window_of_the_inference_script_call():
    """S = 25 (scripts/inference.py:125): model times 999.0, 959.04, ..., 39.96; tau = eta at steps 6-20 (t_5 = 0.8002)."""
    co = so.step_coefficients(25, 1.0)
    times = [c["t_input"] for c in co]
    assert round(times[0], 2) == 999.0 and round(times[1], 2) == 959.04 and round(times[-1], 2) == 39.96
    stochastic = [i for i, c in enumerate(co) if c["c_noise"] != 0.0]          # corrector of step i uses tau(t_i)
    assert stochastic == list(range(6, 21))
    assert co[-1]["p_noise"] == 0.0 and co[0]["c_x"] == 1.0 and co[0]["p_m1"] == 0.0


@pytest.mark.parametrize("S", [2, 3, 5, 25, 40])
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_product_plan_matches_oracle(S, eta):
    plan = sa_sampler.SASolverSampler(lambda *a, **k: None).plan(S, eta)
    want = so.step_coefficients(S, eta)
    assert len(plan) == len(want) == S
    for p, w in zip(plan, want):
        assert set(p) == set(w)
        for k in w:
            assert abs(p[k] - w[k]) <= 1e-6 * max(1.0, abs(w[k])), (k, p[k], w[k])


def test_sa_step_struct_matches_header_size():
    src = '#include <stdio.h>\n#include "pixart_sm100.h"\nint main(){printf("%zu\\n", sizeof(PxaSaStepArgs));return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        size = int(subprocess.check_output([os.path.join(d, "s")]))
    assert size == ctypes.sizeof(lib.SaStepArgs)


def test_sampler_rejects_cpu_tensors_and_unsupported_arguments():
    s = sa_sampler.SASolverSampler(lambda *a, **k: None)
    cond = torch.zeros(1, 1, 2, 2)
    kw = dict(S=4, batch_size=1, shape=(4, 8, 8), conditioning=cond, unconditional_conditioning=cond,
              unconditional_guidance_scale=4.5)
    with pytest.raises(RuntimeError, match="no CPU path"):
        s.sample(**kw, x_T=torch.zeros(1, 4, 8, 8))
    with pytest.raises(RuntimeError, match="no CPU path"):
        sa_sampler.SASolverSampler(lambda *a, **k: None, device="cpu").sample(**kw)
    for bad in (dict(mask=torch.ones(1)), dict(x0=torch.zeros(1)), dict(quantize_x0=True), dict(score_corrector=object()),
                dict(normals_sequence=[]), dict(noise_dropout=0.1), dict(temperature=0.9)):
        with pytest.raises(NotImplementedError):
            s.sample(**kw, **bad)
    with pytest.raises(NotImplementedError):
        s.sample(**dict(kw, conditioning={"c_crossattn": [cond]}))
    with pytest.raises(NotImplementedError):
        sa_sampler.SASolverSampler(lambda *a, **k: None, noise_schedule="squaredcos_cap_v2")
    with pytest.raises(ValueError):
        s.plan(1, 1.0)


@pytest.mark.skipif(not refshim.reference_available(), reason="reference checkout not present")
def test_install_into_reference_repoints_sa_solver_sampler():
    """After install_into_reference(), `from diffusion import SASolverSampler` (scripts/inference.py:19) is the native sampler,
    and inference.py's constructor call (:123) builds against it."""
    refshim.install_reference_shims()
    import pixart_sigma_b200
    assert pixart_sigma_b200.install_into_reference()
    import diffusion
    from diffusion import SASolverSampler
    assert SASolverSampler is sa_sampler.SASolverSampler and diffusion.SASolverSampler is sa_sampler.SASolverSampler
    m = pixart_sigma_b200.PixArtMS(depth=1, input_size=32, model_max_length=300)
    solver = SASolverSampler(m.forward_with_dpmsolver, device="cuda")
    assert solver.model == m.forward_with_dpmsolver
