"""CPU tests of the LCM sampler and distillation: the oracle (oracle/lcm_oracle.py) against the fixtures written from the
unmodified reference (tests/golden/lcm_*.pt, oracle/gen_golden_lcm.py), the host plans of pixart_sigma_b200.lcm against the
reference's tensors bit for bit, the CPU generator state of the sampler's draws, the C ABI struct sizes and argument checks."""
import ctypes
import os
import subprocess
import sys
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dpm_oracle as do                      # noqa: E402
from oracle import lcm_oracle as lo                      # noqa: E402
from oracle import pixart_oracle as po                   # noqa: E402
from oracle.gen_golden_lcm import DISTILL_CASES, SAMPLER_CASES  # noqa: E402
from oracle.gen_golden_train import fingerprint_positions  # noqa: E402
from pixart_sigma_b200 import lib                        # noqa: E402
from pixart_sigma_b200.lcm import LCMDistiller, LCMSampler, LCMScheduler, distill_table  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _gold(name):
    return torch.load(os.path.join(GOLD, name + ".pt"))


@pytest.mark.parametrize("name", sorted(SAMPLER_CASES))
def test_oracle_sampler_reproduces_reference_fixture(name):
    g = _gold(name)
    model = lambda x, t, **kw: do.toy_model(x, t, g["cond"])
    out, draws = lo.sample(model, g["x_T"].clone(), steps=g["case"]["steps"], noise=g["draws"] if len(g["draws"]) else None)
    assert torch.equal(out, g["out"])
    torch.manual_seed(g["seed"])                          # drawing itself: same draws, same generator state
    out2, draws2 = lo.sample(model, g["x_T"].clone(), steps=g["case"]["steps"])
    assert torch.equal(out2, g["out"]) and torch.equal(draws2, g["draws"])
    assert torch.equal(torch.get_rng_state(), g["rng_after"])


@pytest.mark.parametrize("name", sorted(SAMPLER_CASES))
def test_sampler_host_plan_and_cpu_generator_state_match_reference(name):
    g = _gold(name)
    steps, n, hw = g["case"]["steps"], g["case"]["n"], g["case"]["hw"]
    sch = LCMScheduler()
    assert torch.equal(sch.alphas_cumprod, g["alphas_cumprod"])
    sch.set_timesteps(steps, 50)
    assert torch.equal(sch.timesteps, g["timesteps"])
    plan = LCMSampler(lambda *a, **k: None).plan(steps, 50)
    ac = g["alphas_cumprod"]
    for i, st in enumerate(plan):                         # the reference's float32 scalars, bit for bit
        t = g["timesteps"][i]
        tp = g["timesteps"][i + 1] if i + 1 < steps else t
        cs, co = lo.scalings(t)
        assert st["t"] == int(t)
        assert st["sqrt_alpha"] == float(ac[t].sqrt()) and st["sqrt_beta"] == float((1 - ac[t]).sqrt())
        assert st["c_skip"] == float(cs) and st["c_out"] == float(co)
        if steps > 1:
            assert st["c_prev"] == float(ac[tp].sqrt()) and st["c_noise"] == float((1 - ac[tp]).sqrt())
        else:
            assert (st["c_prev"], st["c_noise"]) == (1.0, 0.0)
    torch.manual_seed(g["seed"])
    draws = LCMSampler.draw_noise(steps, (n, 4) + tuple(hw))
    assert (draws is None) == (steps == 1)
    if draws is not None:
        assert torch.equal(draws, g["draws"])
    assert torch.equal(torch.get_rng_state(), g["rng_after"])


def test_distillation_table_matches_reference_plan():
    g = _gold("lcm_distill_d2")
    plan = g["plan"]
    ts, acp, rows = distill_table(50, 1000)
    assert torch.equal(ts, plan["ddim_timesteps"]) and torch.equal(acp, plan["ddim_alpha_cumprods_prev"])
    assert len(rows) == 50
    sch = lo.Schedule()
    for k, r in enumerate(rows):
        s = int(ts[k])
        t = max(s - 20, 0)
        assert (r["cskip_s"], r["cout_s"]) == tuple(float(v) for v in plan["scalings_start"][:, k])
        assert (r["cskip_t"], r["cout_t"]) == tuple(float(v) for v in plan["scalings_t"][:, k])
        assert r["sqrt_acp"] == float(plan["sqrt_acp"][k]) and r["sqrt_1macp"] == float(plan["sqrt_1macp"][k])
        f32 = lambda arr, i: float(torch.tensor(arr[i]).float())
        assert r["sra_s"] == f32(sch.sqrt_recip_ac, s) and r["srm1_s"] == f32(sch.sqrt_recipm1_ac, s)
        assert r["sra_t"] == f32(sch.sqrt_recip_ac, t) and r["srm1_t"] == f32(sch.sqrt_recipm1_ac, t)
    assert rows[0]["cskip_t"] == 1.0 and rows[0]["cout_t"] == 0.0        # index 0: t clamps to 0


def _replay_models(g):
    pad = lambda e: torch.cat([e, torch.zeros_like(e)], dim=1)
    student = lambda x, t, y, mask: pad(g["eps_s"])
    teacher = lambda x, t, y, mask: pad(g["eps_c"] if y is not None else g["eps_u"])
    ema = lambda x, t, y, mask: pad(g["eps_e"])
    return student, teacher, ema


def test_oracle_distillation_step_reproduces_reference_fixture():
    """The oracle's glue (q_sample, x0 predictions, CFG, fp64 DDIM step, target, both losses) on the reference's own model
    outputs gives the reference's tensors bit for bit."""
    g = _gold("lcm_distill_d2")
    student, teacher, ema = _replay_models(g)
    r = lo.distill_step(student, lambda x, t, y, mask: teacher(x, t, None if y is None else y, mask), ema,
                        _latents(g), y=object(), mask=None, noise=g["noise"], index=g["index"], uncond=None)
    assert torch.equal(r["start"], g["start"]) and torch.equal(r["t"], g["t"])
    assert int(g["t"][0]) == 0 and int(g["index"][0]) == 0
    for k in ("x_t", "model_pred", "x_prev", "target", "loss_huber", "loss_l2"):
        assert r[k].dtype == g[k].dtype and torch.equal(r[k], g[k]), k
    assert g["x_prev"].dtype == torch.float64 and g["target"].dtype == torch.float64


def _latents(g):
    from oracle.gen_golden_train import train_inputs
    cfg = po.OracleConfig(**g["cfg"])
    return train_inputs(cfg, g["batch"], tuple(g["hw"]), [0] * g["batch"], g["lens"])[0]


def test_oracle_ema_update_reproduces_reference_fixture():
    g = _gold("lcm_distill_d2")
    cfg = po.OracleConfig(**g["cfg"])
    src = po.synthetic_state_dict(cfg, seed=g["seeds"]["student"])
    dest = po.synthetic_state_dict(cfg, seed=g["seeds"]["ema"])
    lo.ema_update(dest, src, 0.95)
    for n, fp in g["ema_after"].items():
        flat = dest[n].flatten()
        assert torch.equal(flat[fingerprint_positions(flat.numel())], fp["vals"]), n


def test_struct_sizes_match_header():
    src = ('#include <stdio.h>\n#include "pixart_sm100.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(PxaLcmStepArgs), '
           'sizeof(PxaLcmRow), sizeof(PxaLcmTeacherArgs), sizeof(PxaLcmLossArgs), sizeof(PxaEmaBucket), sizeof(PxaEmaArgs));'
           'return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "s.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        sizes = [int(v) for v in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert sizes == [ctypes.sizeof(lib.LcmStepArgs), ctypes.sizeof(lib.LcmRow), ctypes.sizeof(lib.LcmTeacherArgs),
                     ctypes.sizeof(lib.LcmLossArgs), ctypes.sizeof(lib.EmaBucket), ctypes.sizeof(lib.EmaArgs)]


@pytest.mark.parametrize("kw", [dict(beta_schedule="scaled_linear"), dict(beta_schedule="squaredcos_cap_v2"),
                                dict(prediction_type="v_prediction"), dict(prediction_type="sample"),
                                dict(trained_betas=[0.1] * 1000), dict(rescale_betas_zero_snr=True)])
def test_unsupported_scheduler_options_raise(kw):
    with pytest.raises(NotImplementedError):
        LCMScheduler(**kw)


def test_bad_arguments_are_rejected():
    x = torch.zeros(1, 4, 8, 8)
    with pytest.raises(RuntimeError, match="no CPU path"):
        LCMSampler(lambda *a, **k: None).sample(x)
    sch = LCMScheduler()
    with pytest.raises(ValueError, match="set_timesteps"):
        sch.step(x, 0, 999, x)
    sch.set_timesteps(4, 50)
    with pytest.raises(RuntimeError, match="no CPU path"):
        sch.step(x, 0, 999, x)
    with pytest.raises(lib.PxaError):                     # CPU tensors never reach the library
        lib.lcm_step(x, x, None, x, x, sqrt_alpha=1., sqrt_beta=0., c_skip=0., c_out=1., c_prev=1., c_noise=0.)
    with pytest.raises(lib.PxaError):
        lib.lcm_teacher_target(torch.zeros(2, 8, 8, 8), x, torch.zeros(1, dtype=torch.long), torch.zeros(48, dtype=torch.uint8),
                               x, w=4.5)
    with pytest.raises(NotImplementedError):
        LCMDistiller(None, None, loss_type="l1")
    with pytest.raises(ValueError):
        LCMDistiller(None, None, ema_decay=1.5)
