"""GPU parity tests (-m gpu): the boundary modules (PixArtMSBlock / PixArtMS) on the sm_90a kernels against
 (a) the oracle evaluated in fp32 on the SAME bf16-rounded weights and inputs (isolates kernel error), and
 (b) the committed golden outputs of the unmodified reference (fp32 weights; adds the bf16 weight-rounding floor).

Stated tolerances (normwise rel-err, SURVEY.md H1):
  * PixArtMSBlock on the fp32 residual stream vs (a): 1e-3  -- the north_star bar;
  * whole model vs (a): 1e-2 (28 blocks of bf16-operand MMAs; bf16 output adds 1.7e-3);
  * whole model vs (b): 1e-2 (adds the bf16 weight-rounding floor, 3.7e-3 by the survey's measurement). The
    reference's own bf16 forward is 1.6e-2..4.9e-2 from its fp32 forward because it also rounds the timestep to bf16
    (PixArtMS.py:174); that cast is opt-in here (`round_timestep_to_dtype`) and tested separately.
Measured values are appended to gpurun_out/parity.txt.
"""
import os

import pytest
import torch

from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

if torch.cuda.is_available():
    from pixart_sigma_b200 import PixArtMS, lib


def _log(line):
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "parity.txt"), "a") as f:
        f.write(line + "\n")


def _bf16_round(sd):
    return {k: v.to(torch.bfloat16).float() for k, v in sd.items()}


def _build(cfg: po.OracleConfig, sd):
    kvc = None
    if cfg.kv_sampling is not None:
        kvc = dict(sampling=cfg.kv_sampling, scale_factor=cfg.kv_scale_factor, kv_compress_layer=list(cfg.kv_compress_layer))
    with torch.device("cuda"):
        m = PixArtMS(depth=cfg.depth, hidden_size=cfg.hidden_size, num_heads=cfg.num_heads, input_size=cfg.input_size,
                     pe_interpolation=cfg.pe_interpolation, model_max_length=cfg.model_max_length,
                     micro_condition=cfg.micro_condition, qk_norm=cfg.qk_norm, kv_compress_config=kvc)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and missing == ["pos_embed"]
    return m.to(torch.bfloat16).eval()


def _case_inputs(fix):
    cfg = po.OracleConfig(**fix["cfg"])
    x, t, y, mask = po.synthetic_inputs(cfg, fix["batch"], tuple(fix["hw"]), seed=0, timesteps=fix["t"], lens=fix["lens"])
    di = None
    if fix["micro"]:
        di = {"img_hw": torch.tensor([[256.0, 256.0]]).repeat(fix["batch"], 1),
              "aspect_ratio": torch.tensor([[1.0]]).repeat(fix["batch"], 1)}
    return cfg, x, t, y, mask, di


def _oracle_on_rounded(cfg, sd, x, t, y, mask, di, round_t=False):
    """fp32 oracle on bf16-rounded weights / latents / text features; the timestep stays fp32 (model default)."""
    r = lambda v: v.to(torch.bfloat16).float()
    return po.forward(_bf16_round(sd), cfg, r(x), r(t) if round_t else t, r(y), mask=mask, data_info=di)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("B,hw,lens,sr", [(2, (32, 32), [300, 77], 1), (1, (24, 40), [120], 1), (2, (32, 32), [9, 300], 2)])
def test_block_forward_matches_oracle_1e3(B, hw, lens, sr, fused):
    """PixArtMSBlock on the kernels (fp32 residual stream) vs the oracle block: the 1e-3 bar of the north_star.
    fused: LayerNorm + t2i_modulate inside the QKV / fc1 GEMM epilogues (the model default) vs the stand-alone norm pass."""
    C, N = 1152, hw[0] * hw[1]
    cfg = po.OracleConfig(depth=1, kv_sampling="conv" if sr > 1 else None, kv_scale_factor=sr,
                          kv_compress_layer=[0] if sr > 1 else [])
    sd = po.synthetic_state_dict(cfg, seed=7)
    m = _build(cfg, sd)
    blk = m.blocks[0]
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, N, C, generator=g)
    t0 = torch.randn(B, 6 * C, generator=g) * 0.3
    ycat = (torch.randn(sum(lens), C, generator=g)).to(torch.bfloat16)
    sdr = _bf16_round(sd)
    want = po.block_forward(sdr, "blocks.0", x, ycat.float()[None], t0, lens, hw, 16, cfg.sr_ratio(0), cfg.kv_sampling)
    # fused path on the fp32 stream
    mod = (sdr["blocks.0.scale_shift_table"][None] + t0.view(B, 6, C)).cuda().contiguous()
    kv_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
    kv_off = torch.tensor([sum(lens[:i]) for i in range(B)], dtype=torch.int32, device="cuda")
    x32 = x.reshape(B * N, C).cuda().contiguous()
    ln = None
    if fused:
        from pixart_sigma_b200.model import _LnFusion, _ln_ctx
        u, v, one_plus = _LnFusion([blk]).prepare(t0.view(B, 6, C).cuda(), mod[None], blk._ws)
        ln = _ln_ctx(u, v, one_plus, 0, torch.empty(B * N, 8, 2, device="cuda"))
    with torch.no_grad():
        got = blk.run_kernels(x32, ycat.cuda(), kv_len, kv_off, max(lens), mod, B, N, hw, blk._ws, ln).view(B, N, C).cpu()
    err = po.rel_err(got, want)
    # error of the update the block adds (the residual x dominates the norm of the output)
    upd = po.rel_err(got - x, want - x)
    _log(f"block B={B} hw={hw} lens={lens} sr={sr} fused_ln={fused}: out rel_err={err:.3e} update rel_err={upd:.3e}")
    # 1e-3 on the block output; the KV-compressed variant has one more bf16 rounding stage (conv+LN output feeds the
    # MMAs in bf16) and is held to 1.5e-3
    assert err < (1e-3 if sr == 1 else 1.5e-3)
    # reference call signature (bf16 in/out, packed y, python list of lengths)
    with torch.no_grad():
        got2 = blk(x.to(torch.bfloat16).cuda(), ycat.cuda()[None], t0.to(torch.bfloat16).cuda(), lens, hw)
    assert got2.dtype == torch.bfloat16 and got2.shape == (B, N, C)
    assert po.rel_err(got2.float().cpu(), want) < 6e-3


@pytest.mark.parametrize("sr", [1, 2])
def test_block_fp32_attention_flag_selects_hi_lo_p(sr):
    """`fp32_attention = True` (set by `set_grad_checkpoint` on every submodule, model/utils.py:31-34; read by
    AttentionKVCompress.forward, PixArt_blocks.py:145-147) makes the self-attention take P as bf16 hi + lo terms: the block is
    at least as close to the fp32 oracle as with bf16 P, the self-attention kernel launch count is unchanged, and the
    result differs from the default mode (the flag is not ignored)."""
    B, hw, lens = 2, (32, 32), [300, 77]
    C, N = 1152, hw[0] * hw[1]
    cfg = po.OracleConfig(depth=1, kv_sampling="conv" if sr > 1 else None, kv_scale_factor=sr,
                          kv_compress_layer=[0] if sr > 1 else [])
    sd = po.synthetic_state_dict(cfg, seed=7)
    m = _build(cfg, sd)
    blk = m.blocks[0]
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, N, C, generator=g)
    t0 = torch.randn(B, 6 * C, generator=g) * 0.3
    ycat = (torch.randn(sum(lens), C, generator=g)).to(torch.bfloat16)
    sdr = _bf16_round(sd)
    want = po.block_forward(sdr, "blocks.0", x, ycat.float()[None], t0, lens, hw, 16, cfg.sr_ratio(0), cfg.kv_sampling)
    mod = (sdr["blocks.0.scale_shift_table"][None] + t0.view(B, 6, C)).cuda().contiguous()
    kv_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
    kv_off = torch.tensor([sum(lens[:i]) for i in range(B)], dtype=torch.int32, device="cuda")
    got, launches = {}, {}
    for flag in (False, True):
        for mod_ in m.modules():
            mod_.fp32_attention = flag
        x32 = x.reshape(B * N, C).cuda().contiguous()
        n0 = lib.launch_count()
        with torch.no_grad():
            got[flag] = blk.run_kernels(x32, ycat.cuda(), kv_len, kv_off, max(lens), mod, B, N, hw, blk._ws, None).view(B, N, C).cpu()
        torch.cuda.synchronize()
        launches[flag] = lib.launch_count() - n0
    e0, e1 = po.rel_err(got[False], want), po.rel_err(got[True], want)
    u0, u1 = po.rel_err(got[False] - x, want - x), po.rel_err(got[True] - x, want - x)
    _log(f"block fp32_attention sr={sr}: out rel_err bf16-P {e0:.3e} / hi+lo P {e1:.3e}; update rel_err {u0:.3e} / {u1:.3e}")
    assert launches[True] == launches[False]
    assert not torch.equal(got[True], got[False])
    assert e1 < (1e-3 if sr == 1 else 1.5e-3) and e1 <= e0 * 1.02


CASES = ["d2_nomask", "d2_nonsquare", "d2_kvconv", "d2_kvave", "d2_kvuniform", "d2_kvuniform_every", "d2_micro",
         "d2_emptykeys", "d2_qknorm"]


@pytest.mark.parametrize("name", CASES)
def test_model_depth2_matches_oracle_and_golden(golden_dir, name):
    fix = torch.load(os.path.join(golden_dir, name + ".pt"))
    cfg, x, t, y, mask, di = _case_inputs(fix)
    sd = po.synthetic_state_dict(cfg, seed=0)
    m = _build(cfg, sd)
    m.output_dtype = torch.float32
    with torch.no_grad():
        got = m(x.cuda(), t.cuda(), y.cuda(), mask=None if mask is None else mask.cuda(), data_info=di).float().cpu()
    want = _oracle_on_rounded(cfg, sd, x, t, y, mask, di)
    e_or, e_gold = po.rel_err(got, want), po.rel_err(got, fix["out"])
    _log(f"model {name}: vs oracle(bf16-rounded weights) {e_or:.3e}  vs reference golden (fp32 weights) {e_gold:.3e}")
    assert got.shape == fix["out"].shape and torch.isfinite(got).all()
    assert e_or < 1e-2
    assert e_gold < 1e-2


@pytest.mark.parametrize("name", ["xl2_256_b1_mask77", "xl2_256_b2_ragged"])
def test_model_xl2_256px_matches_oracle_and_golden(golden_dir, name):
    """BASELINE config c1 geometry (PixArt-Sigma-XL/2, 256px) on the GPU kernels."""
    fix = torch.load(os.path.join(golden_dir, name + ".pt"))
    cfg, x, t, y, mask, di = _case_inputs(fix)
    sd = po.synthetic_state_dict(cfg, seed=0)
    m = _build(cfg, sd)
    with torch.no_grad():
        got_bf16 = m(x.cuda(), t.cuda(), y.cuda(), mask=mask.cuda())
        m.output_dtype = torch.float32
        got = m(x.cuda(), t.cuda(), y.cuda(), mask=mask.cuda()).cpu()
    assert got_bf16.dtype == torch.bfloat16 and got_bf16.shape == fix["out"].shape
    want = _oracle_on_rounded(cfg, sd, x, t, y, mask, di)
    e_or, e_gold = po.rel_err(got, want), po.rel_err(got, fix["out"])
    _log(f"model {name}: vs oracle(bf16-rounded weights) {e_or:.3e}  vs reference golden (fp32 weights) {e_gold:.3e}")
    assert e_or < 1e-2
    assert e_gold < 1e-2
    # the reference's bf16 timestep cast, opt-in: 749.25 -> 748 must reproduce the oracle fed the rounded timestep
    m.round_timestep_to_dtype = True
    with torch.no_grad():
        got_r = m(x.cuda(), t.cuda(), y.cuda(), mask=mask.cuda()).cpu()
    m.round_timestep_to_dtype = False
    e_round = po.rel_err(got_r, _oracle_on_rounded(cfg, sd, x, t, y, mask, di, round_t=True))
    _log(f"model {name}: bf16-cast timestep vs oracle with the same cast {e_round:.3e}")
    assert e_round < 1e-2
    # eps half for DPM-Solver, and the CFG wrapper's 3-channel quirk
    with torch.no_grad():
        eps = m.forward_with_dpmsolver(x.cuda(), t.cuda(), y.cuda(), None, mask=mask.cuda())
    assert torch.equal(eps.cpu(), got[:, :4])


def test_arbitrary_zero_one_mask_equals_masked_select_packing():
    """Non-prefix masks: device-side compaction must equal the reference's masked_select packing (PixArtMS.py:200)."""
    cfg = po.OracleConfig(depth=1, input_size=32, pe_interpolation=0.5)
    sd = po.synthetic_state_dict(cfg, seed=3)
    x, t, y, _ = po.synthetic_inputs(cfg, 2, (16, 24), seed=3, timesteps=[749.25, 3.0])
    mask = (torch.rand(2, 300, generator=torch.Generator().manual_seed(5)) > 0.5).long()
    m = _build(cfg, sd)
    m.output_dtype = torch.float32
    with torch.no_grad():
        got = m(x.cuda(), t.cuda(), y.cuda(), mask=mask.cuda()).cpu()
        got_b = m(x.cuda(), t.cuda(), y.cuda(), mask=mask[:1].cuda()).cpu()      # broadcast over the batch (CFG)
    assert po.rel_err(got, _oracle_on_rounded(cfg, sd, x, t, y, mask, None)) < 1e-2
    assert po.rel_err(got_b, _oracle_on_rounded(cfg, sd, x, t, y, mask[:1], None)) < 1e-2


def test_forward_is_deterministic_and_sync_free_inputs_on_host_ok():
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    m = _build(cfg, po.synthetic_state_dict(cfg, seed=1))
    x, t, y, mask = po.synthetic_inputs(cfg, 2, (32, 32), lens=[300, 20])
    with torch.no_grad():
        a = m(x, t, y, mask=mask)          # host tensors are moved by forward, like the reference's .to(self.dtype)
        b = m(x.cuda(), t.cuda(), y.cuda(), mask=mask.cuda())
    assert torch.equal(a, b)


def test_cuda_graph_replay_equals_eager():
    """One whole forward captured as a CUDA graph (no host sync / allocation inside the library) replays bit-exactly."""
    from pixart_sigma_b200.graph import GraphedForward
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    m = _build(cfg, po.synthetic_state_dict(cfg, seed=1))
    gf = GraphedForward(m)
    outs = []
    for seed in (0, 1):
        x, t, y, mask = po.synthetic_inputs(cfg, 2, (32, 32), seed=seed, lens=[300, 20 + seed])
        with torch.no_grad():
            eager = m.forward_with_dpmsolver(x.cuda(), t.cuda(), y.cuda(), None, mask=mask.cuda()).clone()
        got = gf(x, t, y.to(torch.bfloat16), mask).clone()
        assert torch.equal(got, eager)
        outs.append(got)
    assert not torch.equal(outs[0], outs[1])


def test_fp16_checkpoint_is_cast_to_bf16_once_and_keeps_fp16_io():
    """scripts/inference.py:161 loads the model as fp16 (`weight_dtype = torch.float16`): the first forward casts the
    parameters to bf16 in place (with a warning), later calls are silent, outputs stay fp16."""
    import warnings
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    sd = po.synthetic_state_dict(cfg, seed=1)
    x, t, y, mask = po.synthetic_inputs(cfg, 2, (32, 32), lens=[300, 20])
    ref = _build(cfg, sd)
    with torch.no_grad():
        want = ref(x.cuda(), t.cuda(), y.cuda(), mask=mask.cuda()).float()
    with torch.device("cuda"):
        m = PixArtMS(depth=2, input_size=32, pe_interpolation=0.5, model_max_length=300)
    m.load_state_dict(sd, strict=False)
    m = m.half().eval()
    with torch.no_grad(), warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        got = m(x.cuda().half(), t.cuda(), y.cuda().half(), mask=mask.cuda())
        assert any("fp16 parameters cast to bf16" in str(w.message) for w in rec)
    assert got.dtype == torch.float16 and m.dtype == torch.bfloat16
    with torch.no_grad(), warnings.catch_warnings(record=True) as rec2:
        warnings.simplefilter("always")
        got2 = m(x.cuda().half(), t.cuda(), y.cuda().half(), mask=mask.cuda())
        assert not rec2
    assert torch.equal(got, got2)
    assert po.rel_err(got.float(), want) < 1e-2        # fp16-rounded inputs / output on top of the bf16 model


def test_drop_path_scales_the_gated_branches_per_sample():
    """Stochastic depth in training mode (timm DropPath, PixArtMS.py:75,77): per sample the attention / MLP branch is
    dropped or scaled by 1 / keep -- equivalent to scaling gate_msa / gate_mlp, which the oracle block gets through t0."""
    B, hw, lens, C = 4, (16, 16), [300, 77, 5, 120], 1152
    N = hw[0] * hw[1]
    cfg = po.OracleConfig(depth=1)
    sd = po.synthetic_state_dict(cfg, seed=7)
    blk = _build(cfg, sd).blocks[0]
    blk.train()
    blk.drop_path_rate = 0.5
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, N, C, generator=g)
    t0 = torch.randn(B, 6 * C, generator=g) * 0.3
    ycat = torch.randn(sum(lens), C, generator=g).to(torch.bfloat16)
    torch.manual_seed(123)
    with torch.no_grad():
        got = blk(x.cuda(), ycat.cuda()[None], t0.cuda(), lens, hw).float().cpu()
    torch.manual_seed(123)
    m = ((torch.rand(B, 2, device="cuda") < 0.5).float() / 0.5).cpu()             # the draw _drop_path_gates makes
    assert 0 < int((m == 0).sum()) < 2 * B                                         # some branches dropped, some kept
    sdr = _bf16_round(sd)
    tab = sdr["blocks.0.scale_shift_table"]
    t0d = t0.view(B, 6, C).clone()
    t0d[:, 2] = m[:, 0:1] * (tab[2] + t0d[:, 2]) - tab[2]
    t0d[:, 5] = m[:, 1:2] * (tab[5] + t0d[:, 5]) - tab[5]
    want = po.block_forward(sdr, "blocks.0", x, ycat.float()[None], t0d.reshape(B, 6 * C), lens, hw, 16, 1, None)
    assert po.rel_err(got, want) < 1.5e-3
    blk.eval()
    with torch.no_grad():
        got_eval = blk(x.cuda(), ycat.cuda()[None], t0.cuda(), lens, hw).float().cpu()
    want_eval = po.block_forward(sdr, "blocks.0", x, ycat.float()[None], t0, lens, hw, 16, 1, None)
    assert po.rel_err(got_eval, want_eval) < 1.5e-3
