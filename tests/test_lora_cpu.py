"""LoRA adapters (pixart_sigma_b200.lora) without a GPU: target matching, peft's file format, merge / unmerge, rejections."""
import json

import pytest
import torch

from pixart_sigma_b200 import PixArtMS, lora

PEFT_KEYS_GLOBAL = ["pos_embed.proj", "caption_projection.linear_1", "caption_projection.linear_2",
                    "adaln_single.emb.timestep_embedder.linear_1", "adaln_single.emb.timestep_embedder.linear_2",
                    "adaln_single.linear", "proj_out"]
PEFT_KEYS_MICRO = ["adaln_single.emb.resolution_embedder.linear_1", "adaln_single.emb.resolution_embedder.linear_2",
                   "adaln_single.emb.aspect_ratio_embedder.linear_1", "adaln_single.emb.aspect_ratio_embedder.linear_2"]
PEFT_KEYS_BLOCK = ["attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_k", "attn2.to_v",
                   "attn2.to_out.0", "ff.net.0.proj", "ff.net.2"]


def _model(micro=False, depth=2):
    torch.manual_seed(0)
    return PixArtMS(depth=depth, input_size=32, pe_interpolation=0.5, model_max_length=300, micro_condition=micro)


@pytest.mark.parametrize("micro", [False, True])
def test_targets_cover_every_projection(micro):
    """The reference target list, under peft's suffix matching, names every projection of the diffusers transformer
    (`proj_in` matches nothing); nothing else is adapted and every base parameter is frozen."""
    m = _model(micro)
    names = lora.inject_lora(m, 16)
    want = PEFT_KEYS_GLOBAL + (PEFT_KEYS_MICRO if micro else []) + \
        [f"transformer_blocks.{i}.{k}" for i in range(2) for k in PEFT_KEYS_BLOCK]
    assert sorted(names) == sorted(want)
    trainable = {n for n, p in m.named_parameters() if p.requires_grad}
    assert trainable and all(n.endswith((".lora_A", ".lora_B")) for n in trainable)


def test_partial_fused_target_rejected():
    m = _model()
    with pytest.raises(NotImplementedError):
        lora.inject_lora(m, 8, target_modules=["to_q"])
    _assert_untouched(m)


def _assert_untouched(m):
    """A rejected inject / load leaves the model as it was: trainable, and without adapters."""
    assert all(p.requires_grad for p in m.parameters())
    assert getattr(m, "_lora", None) is None and not any(hasattr(x, "lora_A") for x in m.modules())


def test_peft_keys_shapes_and_init():
    m = _model()
    lora.inject_lora(m, 8, generator=torch.Generator().manual_seed(3))
    sd = lora.adapter_state_dict(m)
    p = "base_model.model."
    assert sd[p + "pos_embed.proj.lora_A.weight"].shape == (8, 4, 2, 2)
    assert sd[p + "pos_embed.proj.lora_B.weight"].shape == (1152, 8, 1, 1)
    for n in "qkv":
        assert sd[p + f"transformer_blocks.0.attn1.to_{n}.lora_A.weight"].shape == (8, 1152)
        assert sd[p + f"transformer_blocks.0.attn1.to_{n}.lora_B.weight"].shape == (1152, 8)
    assert sd[p + "transformer_blocks.1.ff.net.2.lora_A.weight"].shape == (8, 4608)
    assert sd[p + "transformer_blocks.1.ff.net.2.lora_B.weight"].shape == (1152, 8)
    assert m.blocks[0].attn.qkv.lora_A.shape == (24, 1152) and m.blocks[0].attn.qkv.lora_B.shape == (3, 1152, 8)
    assert m.blocks[0].cross_attn.kv_linear.lora_B.shape == (2, 1152, 8)
    assert len(sd) == 2 * 27 and all(v.dtype == torch.float32 for v in sd.values())
    # peft's gaussian init: A ~ N(0, (1/r)^2), B = 0
    a = torch.cat([v.flatten() for k, v in sd.items() if "lora_A" in k])
    assert abs(a.std().item() - 1 / 8) < 2e-3 and abs(a.mean().item()) < 2e-3
    assert all((v == 0).all() for k, v in sd.items() if "lora_B" in k)


def test_save_load_roundtrip_bitwise(tmp_path):
    m = _model()
    lora.inject_lora(m, 4, use_rslora=True, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        for mod in m.modules():
            if hasattr(mod, "lora_B"):
                mod.lora_B.normal_()
    lora.save_adapter(m, str(tmp_path))
    cfg = json.loads((tmp_path / "adapter_config.json").read_text())
    assert cfg["peft_type"] == "LORA" and cfg["r"] == 4 and cfg["lora_alpha"] == 8 and cfg["use_rslora"] is True
    assert cfg["init_lora_weights"] == "gaussian" and cfg["lora_dropout"] == 0.0 and cfg["bias"] == "none"
    assert sorted(cfg["target_modules"]) == sorted(lora.TARGET_MODULES)
    m2 = _model()
    lora.load_adapter(m2, str(tmp_path))
    a, b = lora.adapter_state_dict(m), lora.adapter_state_dict(m2)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert m2._lora["scale"] == 8 / 2.0


def _write(tmp_path, m, **cfg_changes):
    lora.save_adapter(m, str(tmp_path))
    cfg = json.loads((tmp_path / "adapter_config.json").read_text())
    cfg.update(cfg_changes)
    (tmp_path / "adapter_config.json").write_text(json.dumps(cfg))


@pytest.mark.parametrize("change,exc", [({"use_dora": True}, NotImplementedError), ({"lora_dropout": 0.1}, NotImplementedError),
                                        ({"bias": "all"}, NotImplementedError), ({"peft_type": "LOHA"}, ValueError),
                                        ({"r": 0}, ValueError), ({"rank_pattern": {"to_q": 4}}, NotImplementedError)])
def test_load_rejects_unsupported_config(tmp_path, change, exc):
    m = _model()
    lora.inject_lora(m, 8)
    _write(tmp_path, m, **change)
    m2 = _model()
    with pytest.raises(exc):
        lora.load_adapter(m2, str(tmp_path))
    _assert_untouched(m2)


def test_load_rejects_mismatched_tensors(tmp_path):
    m = _model()
    lora.inject_lora(m, 8)
    _write(tmp_path, m, target_modules=["to_q", "to_k", "to_v", "proj_out", "to_out.0"])   # file has more tensors
    m2 = _model()
    with pytest.raises(ValueError):
        lora.load_adapter(m2, str(tmp_path))
    _assert_untouched(m2)


def test_load_rejects_wrong_shape(tmp_path):
    from safetensors.torch import load_file, save_file
    m = _model()
    lora.inject_lora(m, 8)
    lora.save_adapter(m, str(tmp_path))
    f = str(tmp_path / "adapter_model.safetensors")
    sd = load_file(f)
    k = "base_model.model.transformer_blocks.0.attn1.to_k.lora_B.weight"
    sd[k] = sd[k][:, :4].contiguous()
    save_file(sd, f)
    m2 = _model()
    with pytest.raises(ValueError, match="to_k"):
        lora.load_adapter(m2, str(tmp_path))
    _assert_untouched(m2)


def test_any_rank_loads(tmp_path):
    """An adapter of any positive rank loads, not only powers of two."""
    m = _model()
    lora.inject_lora(m, 12, generator=torch.Generator().manual_seed(0))
    lora.save_adapter(m, str(tmp_path))
    m2 = _model()
    lora.load_adapter(m2, str(tmp_path))
    assert m2.blocks[0].attn.qkv.lora_A.shape == (36, 1152) and m2._lora["scale"] == 8 / 12


@pytest.mark.parametrize("kw", [dict(use_dora=True), dict(lora_dropout=0.05), dict(bias="lora_only")])
def test_inject_rejects_dora_dropout_bias(kw):
    with pytest.raises(NotImplementedError):
        lora.inject_lora(_model(), 8, **kw)


def test_merge_unmerge(tmp_path):
    """merge: W + s B A computed in fp32, rounded once to the parameter dtype (block-diagonal over the fused qkv); unmerge
    restores every weight bit for bit."""
    m = _model().to(torch.bfloat16)
    lora.inject_lora(m, 16, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        for mod in m.modules():
            if hasattr(mod, "lora_B"):
                mod.lora_B.normal_(std=0.01)
    before = {k: v.clone() for k, v in m.state_dict().items()}
    lora.merge_lora(m)
    s = 8 / 16
    qkv = m.blocks[1].attn.qkv
    A, B = qkv.lora_A.detach(), qkv.lora_B.detach()
    w0 = before["blocks.1.attn.qkv.weight"].float()
    for g in range(3):
        want = (w0[g * 1152:(g + 1) * 1152] + s * (B[g] @ A[g * 16:(g + 1) * 16])).to(torch.bfloat16)
        assert torch.equal(qkv.weight[g * 1152:(g + 1) * 1152], want)
    pe = m.x_embedder.proj
    want = (before["x_embedder.proj.weight"].float() + s * (pe.lora_B[0] @ pe.lora_A.flatten(1)).view(1152, 4, 2, 2)).to(torch.bfloat16)
    assert torch.equal(pe.weight, want)
    assert not torch.equal(m.final_layer.linear.weight, before["final_layer.linear.weight"])
    with pytest.raises(RuntimeError):
        lora.merge_lora(m)
    lora.unmerge_lora(m)
    after = m.state_dict()
    assert all(torch.equal(after[k], v) for k, v in before.items())


def test_forward_with_unmerged_adapter_raises():
    m = _model()
    lora.inject_lora(m, 8)
    with pytest.raises(RuntimeError, match="merge_lora"):
        m(torch.zeros(1, 4, 32, 32), torch.zeros(1), torch.zeros(1, 1, 300, 4096))
    with torch.no_grad(), pytest.raises(RuntimeError, match="merge_lora"):
        m(torch.zeros(1, 4, 32, 32), torch.zeros(1), torch.zeros(1, 1, 300, 4096))


def test_one_adapter_per_model():
    m = _model()
    lora.inject_lora(m, 8)
    with pytest.raises(RuntimeError):
        lora.inject_lora(m, 8)
