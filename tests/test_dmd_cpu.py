"""CPU tests of DMD: the oracle (oracle/dmd_oracle.py) against the fixtures written from the unmodified reference
(tests/golden/dmd_*.pt, oracle/gen_golden_dmd.py), the alphas table, the EMA decay sequence, the draw order, argument
validation, the "no CPU path" errors, the unconditional caption's ids and mask, and the C ABI struct size."""
import ctypes
import os
import subprocess
import sys
import tempfile
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dmd_oracle as dmo                     # noqa: E402
from oracle import dpm_oracle as do                      # noqa: E402
from oracle import pixart_oracle as po                   # noqa: E402
from oracle.gen_golden_dmd import CFG, SAMPLE_CASES, STEP_CASES, step_inputs  # noqa: E402
from oracle.gen_golden_train import fingerprint_positions  # noqa: E402
from pixart_sigma_b200 import lib                        # noqa: E402
from pixart_sigma_b200.dmd import DMDDistiller, DMDSampler, ddpm_alphas_cumprod, dmd_draws, ema_decay, null_caption  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def _gold(name):
    return torch.load(os.path.join(GOLD, name + ".pt"))


def _draws(g):
    """The case's draws, regenerated from its seed (pinned against the reference by test_draw_order_matches_reference)."""
    torch.manual_seed(g["rng"])
    return dmd_draws(2, (CFG["input_size"],) * 2, "cpu")


def _matches(t, fp):
    flat = t.detach().flatten().float()
    return torch.equal(flat[fingerprint_positions(flat.numel())], fp["vals"]) and torch.equal(flat.norm(), fp["norm"])


def test_alphas_cumprod_matches_scheduler_stand_in():
    ac = ddpm_alphas_cumprod()
    assert ac.dtype == torch.float32 and ac.shape == (1000,)
    for name in SAMPLE_CASES:
        assert torch.equal(ac, _gold(name)["alphas_cumprod"])
    assert torch.equal(ac, dmo.alphas_cumprod())


@pytest.mark.parametrize("name", sorted(n for n, c in SAMPLE_CASES.items() if c["model"] == "toy"))
def test_oracle_sampler_reproduces_reference_fixture(name):
    g = _gold(name)
    out = dmo.sample(lambda x, t: do.toy_model(x, t, g["cond"]), g["x_T"], g["case"]["t"])
    assert torch.equal(out, g["out"])


@pytest.mark.parametrize("name", sorted(STEP_CASES))
def test_oracle_loss_glue_reproduces_reference_fixture(name):
    """add_noise, score_real / score_fake, coeff, pred, weight and dm_loss on the reference's own model outputs: bit for bit."""
    g = _gold(name)
    ac = ddpm_alphas_cumprod()
    noisy = dmo.add_noise(ac, g["latents"], _draws(g)[1], g["t"])
    assert torch.equal(noisy, g["noisy"])
    r = dmo.dm_loss(g["latents"], noisy, g["t"], g["real_out"], g["fake_out"], ac, 3.0)
    for k in ("weight", "dm_loss"):
        assert torch.equal(r[k], g[k]), k
    assert _matches(r["coeff"], g["coeff"])
    assert sorted(g["t"].tolist()) == [4, 997]                # drawn near both ends of [1, 999)


def test_oracle_step_matches_reference_fixture():
    """The oracle's whole step through pixart_oracle's model (a restatement, so not bit for bit) against the reference."""
    g = _gold("dmd_step_d2")
    cfg = po.OracleConfig(**CFG)
    sds = {k: {n: v.clone().requires_grad_(k in ("generator", "fake")) for n, v in po.synthetic_state_dict(cfg, seed=s).items()}
           for k, s in g["seeds"].items()}
    net = lambda sd: (lambda x, t, y, m: po.forward_grad(sd, cfg, x, t.float(), y, mask=m))
    y, mask, uy, um = step_inputs(cfg, 2, g["lens"])
    draws = _draws(g)
    r = dmo.step(net(sds["generator"]), net(sds["real"]), net(sds["fake"]), y[:, None], mask, uy[:, None], um, draws)
    r["dm_loss"].backward()
    r["sg_loss"].backward()
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    assert rel(r["latents"].detach(), g["latents"]) < 1e-5
    assert rel(r["weight"], g["weight"]) < 1e-5
    assert abs(float(r["coeff"].norm()) - float(g["coeff"]["norm"])) < 1e-4 * float(g["coeff"]["norm"])
    assert abs(float(r["dm_loss"].detach()) - float(g["dm_loss"])) / float(g["dm_loss"]) < 1e-4
    assert abs(float(r["sg_loss"].detach()) - float(g["sg_loss"])) / float(g["sg_loss"]) < 1e-5
    for which, key in (("generator", "grads_gen"), ("fake", "grads_fake")):
        for n, fp in g[key].items():
            flat = sds[which][n].grad.flatten()
            assert abs(float(flat.norm()) - float(fp["norm"])) <= 1e-3 * float(fp["norm"]) + 1e-12, (which, n)


def test_ema_decay_sequence_and_update():
    g = _gold("dmd_step_d2")
    assert [ema_decay(k + 1) for k in range(len(g["ema_decays"]))] == g["ema_decays"] == [0.0, 2 / 11]
    assert [ema_decay(k) for k in (1, 2, 3, 10)] == [0.0, 2 / 11, 3 / 12, 10 / 19]
    assert ema_decay(10 ** 6) == 0.9999 and ema_decay(10 ** 6, max_decay=0.5) == 0.5
    cfg = po.OracleConfig(**CFG)
    shadow = po.synthetic_state_dict(cfg, seed=g["seeds"]["ema"])
    for k, src in enumerate(("generator", "fake")):
        dmo.ema_step(shadow, po.synthetic_state_dict(cfg, seed=g["seeds"][src]), dmo.ema_decay(k + 1))
    for n, fp in g["ema_after"].items():
        flat = shadow[n].flatten()
        assert torch.equal(flat[fingerprint_positions(flat.numel())], fp["vals"]), n


@pytest.mark.parametrize("name", sorted(STEP_CASES))
def test_draw_order_matches_reference(name):
    g = _gold(name)
    torch.manual_seed(g["rng"])
    init_noise, noise, t, noise_f, t_f = dmd_draws(2, (CFG["input_size"],) * 2, "cpu")
    for a, k in ((init_noise, "init_noise"), (noise, "noise"), (noise_f, "noise_for_fake")):
        assert a.shape == (2, 4, CFG["input_size"], CFG["input_size"]) and _matches(a, g["draws"][k]), k
    for a, k in ((t, "t"), (t_f, "t_f")):
        assert a.dtype == g[k].dtype and torch.equal(a, g[k]), k
    assert torch.equal(torch.get_rng_state(), g["rng_after"])
    torch.manual_seed(0)
    fixed = dmd_draws(2, (8, 8), "cpu", fix_noise_ts=500)
    assert fixed[2].tolist() == [500, 500] and fixed[4].tolist() == [500, 500]


def test_null_caption_ids_and_mask():
    seen = {}

    def t5(ids, attention_mask=None):
        seen["ids"], seen["mask"] = ids, attention_mask
        return {"last_hidden_state": torch.ones(ids.shape[0], ids.shape[1], 16)}
    y, mask = null_caption(t5, 120)
    assert seen["ids"].tolist() == [[1] + [0] * 119] and seen["mask"].tolist() == [[1] + [0] * 119]
    assert y.shape == (1, 1, 120, 16) and torch.equal(mask, seen["mask"])


def _stub(prob=0.0):
    return types.SimpleNamespace(y_embedder=types.SimpleNamespace(uncond_prob=prob))


def test_argument_validation():
    uy, um = torch.zeros(1, 8, 16), torch.ones(1, 8)
    with pytest.raises(NotImplementedError, match="use_regression"):
        DMDDistiller(_stub(), None, _stub(), None, uy, um, use_regression=True)
    with pytest.raises(NotImplementedError, match="snr_gamma"):
        DMDDistiller(_stub(), None, _stub(), None, uy, um, snr_gamma=5.0)
    with pytest.raises(NotImplementedError, match="noise_offset"):
        DMDDistiller(_stub(), None, _stub(), None, uy, um, noise_offset=0.1)
    with pytest.raises(ValueError, match="class_dropout_prob"):
        DMDDistiller(_stub(0.1), None, _stub(), None, uy, um)
    with pytest.raises(ValueError, match="class_dropout_prob"):
        DMDDistiller(_stub(), None, _stub(0.1), None, uy, um)
    for kw in (dict(one_step_t=1000), dict(start_ts=1), dict(fix_noise_ts=-1), dict(ema_max_decay=1.5)):
        with pytest.raises(ValueError):
            DMDDistiller(_stub(), None, _stub(), None, uy, um, **kw)
    with pytest.raises(ValueError, match="one caption"):
        DMDDistiller(_stub(), None, _stub(), None, torch.zeros(2, 8, 16), um)
    with pytest.raises(ValueError, match="uncond_mask"):
        DMDDistiller(_stub(), None, _stub(), None, uy, torch.ones(1, 7))
    with pytest.raises(ValueError):
        DMDSampler(lambda *a, **k: None, timestep=1000)


def test_no_cpu_path():
    x = torch.zeros(2, 4, 8, 8)
    with pytest.raises(RuntimeError, match="no CPU path"):
        DMDSampler(lambda *a, **k: None).sample(x)
    with pytest.raises(lib.PxaError):                     # CPU tensors never reach the library
        lib.dmd_loss(x, x, torch.zeros(2, dtype=torch.long), ddpm_alphas_cumprod(), torch.zeros(4, 8, 8, 8),
                     torch.zeros(2, 8, 8, 8), torch.zeros(2, 8, 8, 8), torch.zeros(()), torch.zeros(2),
                     torch.zeros(2 * 2 * lib.DMD_PARTS, dtype=torch.float64), cfg=3.0, gen_sqrt_alpha=1.0, gen_sqrt_beta=0.0)


def test_struct_size_matches_header():
    src = '#include <stdio.h>\n#include "pixart_sm100.h"\nint main(){printf("%zu %d\\n", sizeof(PxaDmdLossArgs), PXA_DMD_PARTS);return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "s.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        size, parts = (int(v) for v in subprocess.check_output([os.path.join(d, "s")]).split())
    assert size == ctypes.sizeof(lib.DmdLossArgs) and parts == lib.DMD_PARTS
