"""CPU tests of pixart_sigma_b200/capture.py: the key that decides when a captured sampling loop may be replayed, the
[uncond ; cond] cache and the step kernels' view of the denoiser output."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pixart_sigma_b200 import PixArtMS                               # noqa: E402
from pixart_sigma_b200.capture import CfgCond, denoiser_key, step_input  # noqa: E402
from pixart_sigma_b200.model import _LnFusion                        # noqa: E402


def _toy(x, t, c, **kw):
    return x


def _kwargs(n=2):
    """model_kwargs as the pipeline passes them: a data_info dict of tensors, plus nested lists and tuples."""
    return dict(mask=torch.ones(n, 8, dtype=torch.long), cfg_scale=4.5,
                data_info={"img_hw": torch.tensor([[256.0, 256.0]]).repeat(n, 1), "aspect_ratio": torch.ones(n, 1),
                           "extra": [torch.zeros(3), (torch.arange(4), "tag")]})


def _clone(obj):
    if isinstance(obj, torch.Tensor):
        return obj.clone()
    if isinstance(obj, dict):
        return {k: _clone(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_clone(v) for v in obj)
    return obj


def _clone_at(obj, path):
    """`obj` with the tensor at `path` (keys / indices) replaced by a clone; everything else is shared."""
    if not path:
        return obj.clone()
    head, rest = path[0], path[1:]
    if isinstance(obj, dict):
        return {k: _clone_at(v, rest) if k == head else v for k, v in obj.items()}
    return type(obj)(_clone_at(v, rest) if i == head else v for i, v in enumerate(obj))


def _model():
    return PixArtMS(depth=1, input_size=32, model_max_length=8).eval()


def test_nested_tensors_are_keyed_by_address_not_value():
    kw = _kwargs()
    key = denoiser_key(_toy, kw)
    assert denoiser_key(_toy, dict(kw)) == key                        # the same tensors in a new dict
    same_values = _clone(kw)
    assert torch.equal(same_values["data_info"]["img_hw"], kw["data_info"]["img_hw"])
    assert denoiser_key(_toy, same_values) != key
    for path in (("data_info", "img_hw"), ("data_info", "extra", 0), ("data_info", "extra", 1, 0)):
        assert denoiser_key(_toy, _clone_at(kw, path)) != key, path  # one equal-valued tensor at a new address
    assert denoiser_key(_toy, dict(kw, cfg_scale=3.0)) != key        # other leaves by value
    assert denoiser_key(_toy, dict(kw, mask=kw["mask"].int())) != key
    assert denoiser_key(lambda *a, **k: None, kw) != key             # another callable


def test_key_never_prints_a_tensor(monkeypatch):
    def refuse(self, *args, **kwargs):
        raise AssertionError("a tensor was printed: its values would be copied to the host")
    monkeypatch.setattr(torch.Tensor, "__repr__", refuse)
    m = _model()
    m.fuse_ln_modulate = True
    kw = _kwargs()
    key = denoiser_key(m.forward_with_dpmsolver, kw)
    assert {key: 1}[denoiser_key(m.forward_with_dpmsolver, kw)] == 1    # hashable, and stable for the same kwargs


def test_output_dtype_and_parameter_dtype_change_the_key():
    m = _model()
    kw = _kwargs()
    key = denoiser_key(m.forward_with_dpmsolver, kw)
    assert denoiser_key(m.forward_with_dpmsolver, kw) == key
    assert denoiser_key(m.forward_with_cfg, kw) != key                # another function of the same module
    m.output_dtype = torch.float32
    k_out = denoiser_key(m.forward_with_dpmsolver, kw)
    assert k_out != key
    m.to(torch.bfloat16)
    assert denoiser_key(m.forward_with_dpmsolver, kw) != k_out
    assert denoiser_key(m, kw) != denoiser_key(_model(), kw)           # a module called directly: by identity


def test_fused_model_key_does_not_depend_on_the_lazily_built_tables():
    m = _model()
    m.fuse_ln_modulate = True
    kw = _kwargs()
    before = denoiser_key(m.forward_with_dpmsolver, kw)
    assert m._ln_fusion is None
    m.__dict__["_ln_fusion"] = _LnFusion(m.blocks)                    # what the first fused forward builds
    assert denoiser_key(m.forward_with_dpmsolver, kw) == before
    with torch.no_grad():
        m.blocks[0].attn.qkv.weight.add_(1.0)                         # the derived tables would be stale: a new key
    assert denoiser_key(m.forward_with_dpmsolver, kw) != before


def test_unfused_model_key_ignores_in_place_weight_updates():
    m = _model()
    kw = _kwargs()
    key = denoiser_key(m.forward_with_dpmsolver, kw)
    with torch.no_grad():
        m.blocks[0].attn.qkv.weight.add_(1.0)                         # a replay reads the weights in place
    assert denoiser_key(m.forward_with_dpmsolver, kw) == key


def test_cfg_cond_is_built_once_and_rebuilt_when_an_input_changes():
    cfg_cond = CfgCond()
    uncond, cond = torch.zeros(1, 1, 4, 8), torch.ones(1, 1, 4, 8)
    first = cfg_cond(uncond, cond)
    assert torch.equal(first, torch.cat([uncond, cond])) and cfg_cond(uncond, cond) is first
    cond.mul_(2)
    second = cfg_cond(uncond, cond)
    assert second is not first and torch.equal(second, torch.cat([uncond, cond]))
    assert cfg_cond(uncond, cond.clone()) is not second


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16, torch.float64])
def test_step_input_keeps_what_the_kernels_read(dtype):
    full = torch.randn(2, 8, 6, 5).to(dtype)
    out = full[:, :4]                                                # a channel slice: dense (h, w) planes
    got = step_input(out)
    assert got.dtype == (dtype if dtype in (torch.float32, torch.bfloat16) else torch.float32)
    assert torch.equal(got, out.to(got.dtype))
    if dtype in (torch.float32, torch.bfloat16):
        assert got.data_ptr() == out.data_ptr()
    assert step_input(out, fp16=True).dtype == (torch.float16 if dtype == torch.float16 else got.dtype)
    strided = full[:, :, :, :4]                                      # (h, w) planes not dense: copied
    assert step_input(strided).is_contiguous()
