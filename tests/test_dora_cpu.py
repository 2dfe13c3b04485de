"""DoRA adapters without a GPU: the DoRA oracle (tests/dora_oracle.py) against its defining properties, peft's file format,
rejections, merge / unmerge, the fp32 glue and the C structs."""
import ctypes
import json
import os
import subprocess
import tempfile

import pytest
import torch
import torch.nn.functional as F

import dora_oracle as do
from oracle import lora_oracle as lo
from oracle import pixart_oracle as po
from pixart_sigma_b200 import PixArtMS, lib, lora

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = "base_model.model."


def _model(depth=2):
    """A model whose weights are all non-zero (the initialisation zeroes the final layer, a zero-norm row for DoRA)."""
    torch.manual_seed(0)
    m = PixArtMS(depth=depth, input_size=32, pe_interpolation=0.5, model_max_length=300)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(std=0.02)
    return m


def _assert_untouched(m):
    assert all(p.requires_grad for p in m.parameters())
    assert getattr(m, "_lora", None) is None and not any(hasattr(x, "lora_A") for x in m.modules())


def _randomize(m, std=0.02, seed=0):
    """Non-zero B and a magnitude away from ||W||, so that c != 1."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for _, mod in lora._adapted(m):
            mod.lora_B.copy_(torch.randn(mod.lora_B.shape, generator=g) * std)
            if hasattr(mod, "lora_magnitude"):
                mod.lora_magnitude.mul_(1 + 0.1 * torch.randn(mod.lora_magnitude.shape, generator=g))


# ------------------------------------------------------------------------------------------------- the oracle
def _layer(seed=0, N=12, K=10, r=3, G=2, dt=torch.float64):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(N, K, generator=g, dtype=dt)
    b = torch.randn(N, generator=g, dtype=dt)
    A = torch.randn(G * r, K, generator=g, dtype=dt) / r
    B = torch.randn(G, N // G, r, generator=g, dtype=dt) * 0.1
    m = W.norm(dim=1) * (1 + 0.1 * torch.randn(N, generator=g, dtype=dt))
    x = torch.randn(7, K, generator=g, dtype=dt)
    return W, b, A, B, m, x


def test_oracle_zero_b_is_the_base_layer():
    W, b, A, B, _, x = _layer()
    m = W.norm(dim=1)
    got = do.dora_linear(x, W, b, A, torch.zeros_like(B), m, 0.5)
    assert torch.allclose(got, F.linear(x, W, b), rtol=0, atol=1e-13)
    wc = torch.randn(6, 4, 2, 2, dtype=torch.float64)
    xc = torch.randn(2, 4, 8, 8, dtype=torch.float64)
    Ac, Bc = torch.randn(3, 4, 2, 2, dtype=torch.float64), torch.zeros(1, 6, 3, dtype=torch.float64)
    got = do.dora_conv(xc, wc, None, Ac, Bc, wc.flatten(1).norm(dim=1), 2.0, 2)
    assert torch.allclose(got, F.conv2d(xc, wc, None, 2), rtol=0, atol=1e-13)


def test_oracle_is_c_times_the_lora_layer_and_the_merge():
    """peft's form base + (c - 1) x W^T + c s lora equals c (x W^T + s lora) + b, and x W_merged^T + b in fp64."""
    W, b, A, B, m, x = _layer()
    s = 0.5
    got = do.dora_linear(x, W, b, A, B, m, s)
    c = m / (W + do.delta(W, A, B, s)).norm(dim=1)
    assert torch.allclose(got, c * (F.linear(x, W) + lo.lora_linear(x, A, B, s)) + b, rtol=1e-12, atol=1e-12)
    merged = do.merged_state_dict({"p.weight": W}, {"p": (A, B, m)}, s)["p.weight"]
    assert torch.allclose(got, F.linear(x, merged, b), rtol=1e-12, atol=1e-12)


def test_oracle_model_unmerged_equals_merged_fp64():
    cfg = po.OracleConfig(depth=1, input_size=16, pe_interpolation=0.5)
    sd = {k: v.double() for k, v in po.synthetic_state_dict(cfg, seed=1).items()}
    g = torch.Generator().manual_seed(2)
    ad = {}
    for name in ("x_embedder.proj", "t_block.1", "blocks.0.attn.qkv", "blocks.0.cross_attn.kv_linear", "blocks.0.mlp.fc2",
                 "final_layer.linear"):
        w = sd[name + ".weight"]
        G = {"blocks.0.attn.qkv": 3, "blocks.0.cross_attn.kv_linear": 2}.get(name, 1)
        A = torch.randn((G * 4,) + tuple(w.shape[1:]), generator=g, dtype=torch.float64) / 4
        B = torch.randn(G, w.shape[0] // G, 4, generator=g, dtype=torch.float64) * 0.02
        m = w.flatten(1).norm(dim=1) * (1 + 0.1 * torch.randn(w.shape[0], generator=g, dtype=torch.float64))
        ad[name] = (A, B, m)
    x, t, y, mask = po.synthetic_inputs(cfg, 1, (16, 16), lens=[20])
    x, y = x.double(), y.double()
    un = do.forward(sd, ad, 2.0, cfg, x, t, y, mask=mask, dtype=torch.float64)
    mg = po.forward(do.merged_state_dict(sd, ad, 2.0), cfg, x, t, y, mask=mask, dtype=torch.float64)
    assert po.rel_err(un, mg) < 1e-12
    base = po.forward(sd, cfg, x, t, y, mask=mask, dtype=torch.float64)
    assert po.rel_err(un, base) > 1e-3


def test_oracle_magnitude_gradient_is_analytic_and_the_norm_is_detached():
    W, b, A, B, m, x = _layer()
    s = 0.5
    A, B, m = (v.clone().requires_grad_() for v in (A, B, m))
    g = torch.randn(7, W.shape[0], dtype=torch.float64)
    (do.dora_linear(x, W, b, A, B, m, s) * g).sum().backward()
    wn = (W + do.delta(W, A.detach(), B.detach(), s)).norm(dim=1)
    z = F.linear(x, W) + lo.lora_linear(x, A.detach(), B.detach(), s)
    assert torch.allclose(m.grad, (g * z).sum(0) / wn, rtol=1e-12, atol=1e-12)
    # dA, dB: autograd of c z + b with c a constant (wn not differentiated)
    A2, B2 = A.detach().clone().requires_grad_(), B.detach().clone().requires_grad_()
    ((m.detach() / wn) * (F.linear(x, W) + lo.lora_linear(x, A2, B2, s)) * g).sum().backward()
    assert torch.allclose(A.grad, A2.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(B.grad, B2.grad, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------- host logic
def test_peft_keys_shapes_and_config(tmp_path):
    m = _model()
    names = lora.inject_dora(m, 8, generator=torch.Generator().manual_seed(3))
    sd = lora.adapter_state_dict(m)
    assert len(sd) == 3 * len(names)
    assert sd[P + "pos_embed.proj.lora_magnitude_vector"].shape == (1, 1152, 1, 1)
    for n in "qkv":
        assert sd[P + f"transformer_blocks.0.attn1.to_{n}.lora_magnitude_vector"].shape == (1152,)
    assert sd[P + "transformer_blocks.1.ff.net.0.proj.lora_magnitude_vector"].shape == (4608,)
    assert m.blocks[0].attn.qkv.lora_magnitude.shape == (3456,) and m.blocks[0].cross_attn.kv_linear.lora_magnitude.shape == (2304,)
    # the magnitude starts at ||W||_row (fp32), on each fused slice
    w = m.blocks[0].attn.qkv.weight.detach()
    assert torch.equal(sd[P + "transformer_blocks.0.attn1.to_k.lora_magnitude_vector"], w[1152:2304].norm(dim=1))
    assert torch.equal(sd[P + "pos_embed.proj.lora_magnitude_vector"].flatten(), m.x_embedder.proj.weight.detach().flatten(1).norm(dim=1))
    trainable = {n for n, p in m.named_parameters() if p.requires_grad}
    assert all(n.endswith((".lora_A", ".lora_B", ".lora_magnitude")) for n in trainable)
    lora.save_adapter(m, str(tmp_path))
    cfg = json.loads((tmp_path / "adapter_config.json").read_text())
    assert cfg["use_dora"] is True and cfg["peft_type"] == "LORA" and cfg["r"] == 8


def test_save_load_roundtrip_bitwise(tmp_path):
    m = _model()
    lora.inject_dora(m, 4, use_rslora=True, generator=torch.Generator().manual_seed(1))
    _randomize(m)
    lora.save_adapter(m, str(tmp_path))
    m2 = _model()
    lora.load_dora_adapter(m2, str(tmp_path))
    a, b = lora.adapter_state_dict(m), lora.adapter_state_dict(m2)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert m2._lora["dora"] and m2._lora["scale"] == 8 / 2.0


def _edit_file(tmp_path, fn):
    from safetensors.torch import load_file, save_file
    f = str(tmp_path / "adapter_model.safetensors")
    sd = load_file(f)
    fn(sd)
    save_file(sd, f)


def _dora_file(tmp_path):
    m = _model()
    lora.inject_dora(m, 8)
    lora.save_adapter(m, str(tmp_path))


K_MAG = P + "transformer_blocks.0.attn1.to_k.lora_magnitude_vector"


@pytest.mark.parametrize("case", ["missing", "extra", "shape", "conv_shape"])
def test_load_rejects_bad_magnitudes(tmp_path, case):
    _dora_file(tmp_path)

    def edit(sd):
        if case == "missing":
            del sd[K_MAG]
        elif case == "extra":
            sd[P + "transformer_blocks.0.attn1.to_k.lora_magnitude_vector2"] = sd[K_MAG].clone()
        elif case == "shape":
            sd[K_MAG] = sd[K_MAG][:1000].contiguous()
        else:
            k = P + "pos_embed.proj.lora_magnitude_vector"
            sd[k] = sd[k].flatten().contiguous()
    _edit_file(tmp_path, edit)
    m2 = _model()
    with pytest.raises(ValueError):
        lora.load_dora_adapter(m2, str(tmp_path))
    _assert_untouched(m2)


def test_lora_file_is_rejected_by_load_dora_adapter_and_dora_file_by_load_adapter(tmp_path):
    m = _model()
    lora.inject_lora(m, 8)
    lora.save_adapter(m, str(tmp_path / "lora"))
    m2 = _model()
    with pytest.raises(ValueError, match="load_adapter"):
        lora.load_dora_adapter(m2, str(tmp_path / "lora"))
    _assert_untouched(m2)
    # a LoRA file relabelled use_dora: its magnitudes are missing
    cfg = json.loads((tmp_path / "lora" / "adapter_config.json").read_text())
    cfg["use_dora"] = True
    (tmp_path / "lora" / "adapter_config.json").write_text(json.dumps(cfg))
    with pytest.raises(ValueError, match="missing"):
        lora.load_dora_adapter(m2, str(tmp_path / "lora"))
    _assert_untouched(m2)
    _dora_file(tmp_path / "dora")
    with pytest.raises(NotImplementedError, match="load_dora_adapter"):
        lora.load_adapter(m2, str(tmp_path / "dora"))
    _assert_untouched(m2)


def test_inject_lora_with_use_dora_names_inject_dora():
    with pytest.raises(NotImplementedError, match="inject_dora"):
        lora.inject_lora(_model(), 8, use_dora=True)


def test_zero_norm_row_raises_and_leaves_the_model_untouched():
    m = _model()
    with torch.no_grad():
        m.blocks[1].mlp.fc2.weight[5].zero_()
    with pytest.raises(ValueError, match="blocks.1.mlp.fc2"):
        lora.inject_dora(m, 4)
    _assert_untouched(m)


def test_merge_unmerge():
    """merge: c (W + s B A) in fp32 with c = m / ||W + s B A||_row, rounded once; unmerge restores every weight bit for bit."""
    m = _model().to(torch.bfloat16)
    lora.inject_dora(m, 16, generator=torch.Generator().manual_seed(2))
    _randomize(m, std=0.01)
    before = {k: v.clone() for k, v in m.state_dict().items()}
    lora.merge_lora(m)
    s = 8 / 16
    for mod, name in ((m.blocks[1].attn.qkv, "blocks.1.attn.qkv"), (m.x_embedder.proj, "x_embedder.proj"),
                      (m.final_layer.linear, "final_layer.linear")):
        w0 = before[name + ".weight"].float()
        A, B, mag = mod.lora_A.detach().float(), mod.lora_B.detach().float(), mod.lora_magnitude.detach().float()
        new = w0 + do.delta(w0, A, B, s)
        c = mag / new.flatten(1).norm(dim=1)
        want = (c.view((-1,) + (1,) * (w0.dim() - 1)) * new).to(torch.bfloat16)
        assert torch.equal(mod.weight, want), name
    lora.unmerge_lora(m)
    after = m.state_dict()
    assert all(torch.equal(after[k], v) for k, v in before.items())


def test_fp32_glue_fresh_adapter_is_bitwise_base_and_matches_oracle():
    m = _model()
    lora.inject_dora(m, 4, generator=torch.Generator().manual_seed(0))
    x = torch.randn(3, 1152)
    xc = torch.randn(2, 4, 16, 16)
    fl, pe = m.final_layer.linear, m.x_embedder.proj
    assert torch.equal(lora.linear_fp32(fl, x), F.linear(x, fl.weight, fl.bias))
    assert torch.equal(lora.conv_fp32(pe, xc), F.conv2d(xc, pe.weight, pe.bias, stride=pe.stride))
    _randomize(m)
    for mod, got, want in (
            (fl, lora.linear_fp32(fl, x), do.dora_linear(x, fl.weight, fl.bias, fl.lora_A, fl.lora_B, fl.lora_magnitude, 2.0)),
            (pe, lora.conv_fp32(pe, xc), do.dora_conv(xc, pe.weight, pe.bias, pe.lora_A, pe.lora_B, pe.lora_magnitude, 2.0,
                                                      pe.stride))):
        assert po.rel_err(got.detach(), want.detach()) < 1e-6
    # the magnitude receives a gradient through the glue, the norm does not
    lora.linear_fp32(fl, x).sum().backward()
    assert fl.lora_magnitude.grad is not None and fl.weight.grad is None


def test_dora_structs_match_the_header():
    """The new ctypes structs against the header compiled with gcc: size and every field offset."""
    structs = {"DoraNormItem": lib.DoraNormItem, "DoraNormArgs": lib.DoraNormArgs, "DoraBwdArgs": lib.DoraBwdArgs}
    want, probes = {}, []
    for name, s in structs.items():
        want[name] = ctypes.sizeof(s)
        probes.append(f'printf("{name} %zu\\n", sizeof(Pxa{name}));')
        for f in s._fields_:
            want[f"{name}.{f[0]}"] = getattr(s, f[0]).offset
            probes.append(f'printf("{name}.{f[0]} %zu\\n", offsetof(Pxa{name}, {f[0]}));')
    probes.append('printf("ROWS %d\\n", PXA_DORA_BWD_ROWS);')
    want["ROWS"] = lib.DORA_BWD_ROWS
    src = '#include <stddef.h>\n#include <stdio.h>\n#include "pixart_sm100.h"\nint main(void) {\n' + "\n".join(probes) + "\nreturn 0;\n}\n"
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "s.c"), "-o", os.path.join(d, "s")])
        got = {k: int(v) for k, v in (line.split() for line in subprocess.check_output([os.path.join(d, "s")], text=True).splitlines())}
    assert got == want
    for name in ("pxa_gemm_dora_bf16", "pxa_dora_norm", "pxa_dora_bwd"):
        assert name in lib.EXPORTS and hasattr(lib.load(), name)
