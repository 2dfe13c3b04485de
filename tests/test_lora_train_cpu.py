"""LoRA training without a GPU: the oracle's LoRA layers, the adapter operands of the kernels, DDPMEpsLoss and the C ABI of
the GEMM K-tail."""
import ctypes
import os
import subprocess
import tempfile

import pytest
import torch

from oracle import lora_oracle as lo
from oracle import pixart_oracle as po
from pixart_sigma_b200 import PixArtMS, lib, lora
from pixart_sigma_b200.dmd import ddpm_alphas_cumprod
from pixart_sigma_b200.training import DDPMEpsLoss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = po.OracleConfig(depth=1, input_size=16, pe_interpolation=0.5, model_max_length=8)


def _adapters(seed=0, zero_b=False, r=4):
    """A depth-1 native model with a rank-r adapter (random B unless zero_b); its adapters in the oracle's layout, fp64."""
    torch.manual_seed(seed)
    m = PixArtMS(depth=1, input_size=16, pe_interpolation=0.5, model_max_length=8)
    lora.inject_lora(m, r, generator=torch.Generator().manual_seed(seed))
    if not zero_b:
        with torch.no_grad():
            for _, mod in lora._adapted(m):
                mod.lora_B.normal_(0, 0.05)
    ad = {n: (mod.lora_A.detach().double(), mod.lora_B.detach().double()) for n, mod in lora._adapted(m)}
    return m, ad, m._lora["scale"]


def _inputs():
    sd = {k: v.double() for k, v in po.synthetic_state_dict(CFG, seed=3).items()}
    x, t, y, mask = po.synthetic_inputs(CFG, 2, (16, 16), lens=[8, 5])
    return sd, x.double(), t.double(), y.double(), mask


def test_oracle_zero_b_is_the_base_forward():
    _, ad, s = _adapters(zero_b=True)
    sd, x, t, y, mask = _inputs()
    assert torch.equal(lo.forward(sd, ad, s, CFG, x, t, y, mask=mask, dtype=torch.float64),
                       po.forward(sd, CFG, x, t, y, mask=mask, dtype=torch.float64))


def test_oracle_unmerged_equals_merged_fp64():
    """peft's unmerged layers (including the fused qkv / kv groups and the patch-embedding conv) equal the merged weights."""
    _, ad, s = _adapters()
    assert {"x_embedder.proj", "blocks.0.attn.qkv", "blocks.0.cross_attn.kv_linear", "t_block.1"} <= set(ad)
    sd, x, t, y, mask = _inputs()
    got = lo.forward(sd, ad, s, CFG, x, t, y, mask=mask, dtype=torch.float64)
    want = po.forward(lo.merged_state_dict(sd, ad, s), CFG, x, t, y, mask=mask, dtype=torch.float64)
    base = po.forward(sd, CFG, x, t, y, mask=mask, dtype=torch.float64)
    assert po.rel_err(got, want) < 1e-12
    assert po.rel_err(got, base) > 1e-3                         # the adapter does move the output


def test_oracle_conv_adapter_is_peft_conv():
    """The patch-embedding adapter: Conv2d(in, r, k, stride) then a 1x1 Conv2d(r, out), against the merged kernel."""
    _, ad, s = _adapters()
    A, B = ad["x_embedder.proj"]
    x = torch.randn(2, 4, 8, 8, dtype=torch.float64)
    got = lo.lora_conv(x, A, B, s, 2)
    want = torch.nn.functional.conv2d(x, s * (B[0] @ A.flatten(1)).view(-1, *A.shape[1:]), stride=2)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


def test_oracle_gradients_reach_the_adapters():
    _, ad, s = _adapters()
    sd, x, t, y, mask = _inputs()
    ad = {k: (a.clone().requires_grad_(), b.clone().requires_grad_()) for k, (a, b) in ad.items()}
    lo.forward_grad(sd, ad, s, CFG, x, t, y, mask=mask, dtype=torch.float64).square().mean().backward()
    assert all(a.grad is not None and b.grad is not None and b.grad.abs().sum() > 0 for a, b in ad.values())


def test_kernel_operands_match_the_parameters():
    """lora.prepare_operands: A padded to T rows, s blockdiag(B), and their transposes, each rounded once to bf16."""
    m, _, s = _adapters(r=4)
    lora.prepare_operands(m)
    qkv = m.blocks[0].attn.qkv
    op = qkv._pxa_lora
    A, B = qkv.lora_A.detach(), qkv.lora_B.detach()
    C = A.shape[1]
    assert op.T == 16 and op.a.shape == (16, C) and op.b.shape == (3 * C, 16)
    a = torch.zeros(16, C)
    a[:12] = A
    bd = torch.zeros(3 * C, 16)
    for g in range(3):
        bd[g * C:(g + 1) * C, g * 4:(g + 1) * 4] = s * B[g]
    for got, want in ((op.a, a), (op.at, a.t()), (op.b, bd), (op.bt, bd.t())):
        assert got.dtype == torch.bfloat16 and torch.equal(got.float(), want.to(torch.bfloat16).float())
    assert not hasattr(m.x_embedder.proj, "_pxa_lora")          # fp32 torch glue: no kernel operands
    lora.merge_lora(m)
    lora.prepare_operands(m)
    assert "_pxa_lora" not in qkv.__dict__                       # a merged adapter is not applied again


def test_ddpm_eps_loss_restates_the_script():
    """noisy = sqrt(a_t) x + sqrt(1 - a_t) noise on the float32 DDPM table; loss = MSE(eps half of the output, noise)."""
    ac = ddpm_alphas_cumprod(1000)
    assert ac.dtype == torch.float32
    x0, noise = torch.randn(3, 4, 8, 8), torch.randn(3, 4, 8, 8)
    t = torch.tensor([0, 500, 999])
    seen = {}

    def model(x_t, timestep, **kw):
        seen["x_t"] = x_t
        return torch.cat([x_t * 0.5, torch.full_like(x_t, 7.0)], 1)

    terms = DDPMEpsLoss().training_losses(model, x0, t, {}, noise=noise)
    a = ac[t].view(-1, 1, 1, 1)
    x_t = a.sqrt() * x0 + (1 - a).sqrt() * noise
    assert torch.equal(seen["x_t"], x_t)
    assert torch.allclose(terms["loss"], ((x_t * 0.5 - noise) ** 2).mean((1, 2, 3)))
    with pytest.raises(NotImplementedError):
        DDPMEpsLoss(snr_gamma=5.0)
    with pytest.raises(NotImplementedError):
        DDPMEpsLoss(prediction_type="v_prediction")


def test_gemm_tail_struct_matches_the_header():
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "pixart_sm100.h"\nint main(){printf("%zu %zu %zu %zu\\n", '
           'sizeof(PxaGemmTail), offsetof(PxaGemmTail, tail_k), offsetof(PxaGemmTail, ldw_tail), sizeof(PxaGemmArgs));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        sizes = [int(v) for v in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert sizes == [ctypes.sizeof(lib.GemmTail), lib.GemmTail.tail_k.offset, lib.GemmTail.ldw_tail.offset,
                     ctypes.sizeof(lib.GemmArgs)]
    assert "pxa_gemm_lora_bf16" in lib.EXPORTS
