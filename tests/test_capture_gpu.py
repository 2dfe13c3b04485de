"""GPU tests (-m gpu) of the captured sampling loops of all five native samplers (pixart_sigma_b200/capture.py): a replay makes
no host sync and reads no buffer freed after the capture, a tensor nested in model_kwargs is captured by address (an
equal-valued one elsewhere captures anew), the denoiser's output dtype is part of the key, and a fused LayerNorm-modulate
PixArtMS replays its first capture.

Graphed and eager loops run the same kernels on the same inputs with replayed draws, so the toy loops must agree bit for bit.
The PixArtMS loops are held to 1e-5, as the existing graphed-loop tests hold them."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pixart_oracle as po         # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SAMPLERS = ["dpm", "sa", "iddpm", "lcm", "dmd"]

if torch.cuda.is_available():
    from pixart_sigma_b200 import PixArtMS, SASolverSampler
    from pixart_sigma_b200.dmd import DMDSampler
    from pixart_sigma_b200.iddpm import IDDPM
    from pixart_sigma_b200.lcm import LCMSampler
    from pixart_sigma_b200.sampler import DPMS


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


class _Toy(torch.nn.Module):
    """A learn-sigma denoiser that reads data_info["shift"][0], a tensor nested in model_kwargs, and has an output_dtype."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.tensor(0.7, device=DEV))
        self.output_dtype = None

    def forward(self, x, timestep, *cond, data_info=None, **kwargs):
        x, tt = x.float(), (timestep.float() / 1000.0).view(-1, 1, 1, 1)
        c = cond[0].float().reshape(cond[0].shape[0], -1).mean(dim=1).view(-1, 1, 1, 1) if cond else 0.0
        eps = torch.tanh(self.w * x + 0.4 * tt + c + data_info["shift"][0])
        return torch.cat([eps, 0.5 * torch.tanh(x)], dim=1).to(self.output_dtype or torch.float32)


def _toy_kwargs(shift=None):
    return {"data_info": {"shift": [torch.full((1, 1, 1, 1), 0.1, device=DEV) if shift is None else shift]}}


def _toy_setup(name, model, kw):
    """(sampler, call(model_kwargs, cuda_graph) -> latents) on 2 x 4 x 8 x 8 latents with replayed draws."""
    g = torch.Generator().manual_seed(0)
    z = torch.randn(2, 4, 8, 8, generator=g).to(DEV)
    cond, uncond = (torch.randn(2, 1, 6, 16, generator=g).to(DEV) for _ in range(2))
    draws = torch.randn(4, 2, 4, 8, 8, generator=g).to(DEV)
    if name == "dpm":                                  # DPMS takes its model_kwargs at construction
        s = DPMS(model, condition=cond, uncondition=uncond, cfg_scale=4.5, model_kwargs=kw)
        return s, lambda kw, graph: s.sample(z, steps=4, cuda_graph=graph)
    if name == "sa":
        s = SASolverSampler(model, device=DEV)
        return s, lambda kw, graph: s.sample(S=4, batch_size=2, shape=(4, 8, 8), eta=1.0, conditioning=cond,
                                             unconditional_conditioning=uncond, unconditional_guidance_scale=4.5,
                                             model_kwargs=kw, x_T=z, noise=list(draws), cuda_graph=graph)[0]
    if name == "iddpm":
        s = IDDPM("4")
        return s, lambda kw, graph: s.p_sample_loop(model, z.shape, z, clip_denoised=False, model_kwargs=kw, device=DEV,
                                                    noise_draws=list(draws), cuda_graph=graph)
    if name == "lcm":
        s = LCMSampler(model)
        return s, lambda kw, graph: s.sample(z, steps=4, model_kwargs=kw, noise=draws, cuda_graph=graph)
    s = DMDSampler(model, timestep=400)
    return s, lambda kw, graph: s.sample(z, model_kwargs=kw, cuda_graph=graph)


@pytest.mark.parametrize("name", SAMPLERS)
def test_replay_has_no_host_sync_and_is_keyed_by_nested_tensor_address_and_output_dtype(name):
    model, kw = _Toy(), _toy_kwargs()
    s, call = _toy_setup(name, model, kw)
    eager = call(kw, False)
    first = call(kw, True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = call(kw, True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert len(s._graphs) == 1 and torch.equal(first, eager) and torch.equal(again, eager)
    # the loop's state stays reserved for its graph: latents-sized buffers allocated after the capture are not the ones a
    # replay reads and writes
    junk = [torch.full_like(eager, float("nan")) for _ in range(16)]
    assert torch.equal(call(kw, True), eager) and all(bool(torch.isnan(j).all()) for j in junk)
    graphs = 1
    if name != "dpm":
        moved = _toy_kwargs(kw["data_info"]["shift"][0].clone())      # equal values at a new address
        got = call(moved, True)
        graphs += 1
        assert len(s._graphs) == graphs and torch.equal(got, call(moved, False)) and torch.equal(got, eager)
    model.output_dtype = torch.bfloat16
    got = call(kw, True)
    assert len(s._graphs) == graphs + 1 and torch.equal(got, call(kw, False)) and not torch.equal(got, eager)


def _pixart_setup(name):
    """(sampler, call(cuda_graph) -> latents) around a depth-2 PixArtMS at 256px (256 tokens) with the fused LayerNorm."""
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    with torch.device(DEV):
        m = PixArtMS(depth=2, input_size=32, pe_interpolation=0.5, model_max_length=300)
    m.load_state_dict(po.synthetic_state_dict(cfg, seed=0), strict=False)
    m = m.to(torch.bfloat16).eval()
    m.fuse_ln_modulate = True
    z, _, y, mask = (v.to(DEV) for v in po.synthetic_inputs(cfg, 1, (32, 32), seed=5, lens=[77]))
    null_y = po.synthetic_inputs(cfg, 1, (32, 32), seed=6)[2].to(DEV)
    draws = torch.randn((2,) + tuple(z.shape), generator=torch.Generator().manual_seed(1)).to(DEV)
    if name == "dpm":
        s = DPMS(m.forward_with_dpmsolver, condition=y, uncondition=null_y, cfg_scale=4.5,
                 model_kwargs=dict(data_info=None, mask=mask))
        return s, lambda graph: s.sample(z, steps=2, cuda_graph=graph)
    if name == "sa":
        s = SASolverSampler(m.forward_with_dpmsolver, device=DEV)
        return s, lambda graph: s.sample(S=2, batch_size=1, shape=(4, 32, 32), eta=1.0, conditioning=y,
                                         unconditional_conditioning=null_y, unconditional_guidance_scale=4.5,
                                         model_kwargs=dict(data_info=None, mask=mask), x_T=z, noise=list(draws),
                                         cuda_graph=graph)[0]
    if name == "iddpm":
        s = IDDPM("2")
        z2, d2 = torch.cat([z, z]), list(torch.cat([draws, draws], dim=1))
        kw = dict(y=torch.cat([y, null_y]), cfg_scale=4.5, data_info=None, mask=mask)
        return s, lambda graph: s.p_sample_loop(m.forward_with_cfg, z2.shape, z2, clip_denoised=False, model_kwargs=kw,
                                                device=DEV, noise_draws=d2, cuda_graph=graph)
    kw = dict(y=y, mask=mask)
    if name == "lcm":
        s = LCMSampler(m)
        return s, lambda graph: s.sample(z, steps=2, model_kwargs=kw, noise=draws, cuda_graph=graph)
    s = DMDSampler(m, timestep=400)
    return s, lambda graph: s.sample(z, model_kwargs=kw, cuda_graph=graph)


@pytest.mark.parametrize("name", SAMPLERS)
def test_fused_layernorm_model_replays_its_first_capture(name):
    """The fused forward builds its weight tables in the first capture's warm-up; the second call must still find that
    capture."""
    s, call = _pixart_setup(name)
    eager = call(False)
    first, second = call(True), call(True)
    assert len(s._graphs) == 1
    assert _rel(first, eager) < 1e-5 and _rel(second, eager) < 1e-5
