"""CPU tests of the native IDDPM loop's host side (pixart_sigma_b200/iddpm.py): the per-step fp32 scalars and mapped timesteps
the step kernel receives, the argument struct against the header, the recognition of the native CFG wrapper, the device
dispatch (CPU latents keep the torch restatement) and the re-pointing of the reference's `diffusion.IDDPM`."""
import ctypes
import os
import subprocess
import sys
import tempfile
import types

import pytest
import torch

from oracle import refshim
from oracle.gen_golden_iddpm import toy_model
from pixart_sigma_b200 import PixArt, PixArtMS, lib
from pixart_sigma_b200 import iddpm as iddpm_mod
from pixart_sigma_b200.iddpm import IDDPM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("respacing", ["10", "100", "4,6,10", "ddim25"])
def test_plan_scalars_and_timesteps_equal_the_torch_restatement(respacing):
    """Every scalar equals what p_mean_variance reads through `_x(name, t)` (the fp64 table entry rounded to fp32), and the
    mapped timestep is `timestep_map[t]`, in sampling order."""
    d = IDDPM(respacing)
    plan = d.plan()
    assert [st["t"] for st in plan] == list(reversed(range(d.num_timesteps)))
    names = {"sqrt_recip_ac": "sqrt_recip_ac", "sqrt_recipm1_ac": "sqrt_recipm1_ac", "post_c1": "post_c1",
             "post_c2": "post_c2", "log_beta": "log_betas", "post_logvar": "post_logvar"}
    for st in plan:
        t = torch.tensor([st["t"]])
        assert st["map_t"] == d.timestep_map[st["t"]]
        for key, name in names.items():
            want = d._x(name, t).flatten()
            assert want.dtype == torch.float32 and torch.equal(torch.tensor([st[key]], dtype=torch.float32), want), (key, st["t"])
    tm = d._timesteps(torch.device("cpu"), 6)
    assert tm.dtype == torch.int64 and tuple(tm.shape) == (d.num_timesteps, 6)
    assert torch.equal(tm[:, 0], torch.tensor([d.timestep_map[i] for i in reversed(range(d.num_timesteps))]))
    assert d._timesteps(torch.device("cpu"), 6) is tm                    # uploaded once


def test_iddpm_step_struct_matches_header():
    src = '#include <stdio.h>\n#include "pixart_sm100.h"\nint main(){printf("%zu %d\\n", sizeof(PxaIddpmStepArgs), PXA_DTYPE_F16);return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        size, f16 = [int(v) for v in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert size == ctypes.sizeof(lib.IddpmStepArgs) and f16 == lib.DTYPE_F16
    assert "pxa_iddpm_step" in lib.EXPORTS


def test_only_the_packages_own_forward_with_cfg_is_mixed_in_the_kernel():
    m = PixArtMS(depth=1, input_size=8, model_max_length=8)
    s = PixArt(depth=1, input_size=8, model_max_length=8)
    assert iddpm_mod._native_cfg_owner(m.forward_with_cfg) is m
    assert iddpm_mod._native_cfg_owner(s.forward_with_cfg) is s
    assert iddpm_mod._native_cfg_owner(m.forward_with_dpmsolver) is None
    assert iddpm_mod._native_cfg_owner(m.forward) is None
    assert iddpm_mod._native_cfg_owner(toy_model()) is None

    class Custom(PixArtMS):                                  # an overridden wrapper is called as it is
        def forward_with_cfg(self, *a, **k):
            return super().forward_with_cfg(*a, **k)
    assert iddpm_mod._native_cfg_owner(Custom(depth=1, input_size=8, model_max_length=8).forward_with_cfg) is None


def test_cpu_latents_take_the_torch_loop(monkeypatch):
    def native(*a, **k):
        raise AssertionError("the native loop ran on CPU latents")
    monkeypatch.setattr(iddpm_mod.IDDPMSampler, "_sample_native", native)
    monkeypatch.setattr(lib, "iddpm_step", native)
    z = torch.randn(2, 4, 6, 5, generator=torch.Generator().manual_seed(0))
    d = IDDPM("7")
    torch.manual_seed(3)
    out = d.p_sample_loop(toy_model(), z.shape, z, clip_denoised=False, model_kwargs=dict(scale=0.9), device="cpu")
    torch.manual_seed(3)
    *_, last = d.p_sample_loop_progressive(toy_model(), z.shape, z, clip_denoised=False, model_kwargs=dict(scale=0.9),
                                           device="cpu")
    assert torch.equal(out, last["sample"])
    with pytest.raises(NotImplementedError):
        d.p_sample_loop(toy_model(), z.shape, z, device="cpu", noise_draws=[torch.zeros_like(z)] * 7)
    with pytest.raises(NotImplementedError):
        d.p_sample_loop(toy_model(), z.shape, z, device="cpu", cuda_graph=True)


def test_training_losses_says_the_native_object_samples_only():
    """train.py's `IDDPM(str(1000), learn_sigma=True, pred_sigma=True, snr=False)` is accepted by the factory, so a training
    script that imports `diffusion.IDDPM` after install_into_reference() gets this object: it must fail with a clear message."""
    d = IDDPM(str(1000), learn_sigma=True, pred_sigma=True, snr=False)
    with pytest.raises(NotImplementedError, match="samples only"):
        d.training_losses(None, torch.zeros(1, 4, 8, 8), torch.zeros(1, dtype=torch.long))


def _check_repointed(steps=20):
    from diffusion import IDDPM as RefIDDPM
    assert RefIDDPM is IDDPM
    got, want = RefIDDPM(str(steps)), IDDPM(str(steps))
    assert type(got) is type(want) and got.timestep_map == want.timestep_map and got.num_timesteps == want.num_timesteps
    assert all((got.tab[k] == want.tab[k]).all() for k in want.tab) and got.plan() == want.plan()
    with pytest.raises(NotImplementedError):
        RefIDDPM(str(steps), predict_xstart=True)


@pytest.mark.skipif(not refshim.reference_available(), reason="/root/reference not present")
def test_install_into_reference_repoints_diffusion_iddpm():
    """scripts/inference.py does `from diffusion import IDDPM` (inference.py:19) and calls `IDDPM(str(sample_steps))`."""
    refshim.install_reference_shims()
    import pixart_sigma_b200
    assert pixart_sigma_b200.install_into_reference()
    _check_repointed()


def test_install_into_reference_repoints_iddpm_in_a_minimal_package(monkeypatch):
    """The same re-pointing against a stand-in `diffusion` package with the module names the hook touches."""
    pkg, model, builder, nets = (types.ModuleType(n) for n in ("diffusion", "diffusion.model", "diffusion.model.builder",
                                                               "diffusion.model.nets"))
    builder.MODELS = types.SimpleNamespace(_module_dict={"PixArtMS": None})
    pkg.model, model.builder, model.nets = model, builder, nets
    for name, mod in (("diffusion", pkg), ("diffusion.model", model), ("diffusion.model.builder", builder),
                      ("diffusion.model.nets", nets)):
        monkeypatch.setitem(sys.modules, name, mod)
    import pixart_sigma_b200
    assert pixart_sigma_b200.install_into_reference()
    assert builder.MODELS._module_dict["PixArtMS"] is PixArtMS
    _check_repointed(steps=100)
