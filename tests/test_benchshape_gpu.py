"""GPU parity tests (-m gpu) AT THE BENCHMARKED GEOMETRIES (BASELINE configs[2..4]; VERDICT r1 "what's weak" 1):

  * one `PixArtMSBlock` at c3 (B=8, N=4096 tokens, ragged caption lengths, M = 32768 GEMM rows) and at c4 (B=2,
    N=16384, KV compression conv sr=2 -> Nk=4096) against the oracle block `po.block_forward` evaluated in fp32 on the
    host on the same bf16-rounded weights -- the north_star's 1e-3 bar (1.5e-3 with KV compression);
  * `pxa_flash_attn_d72_bf16` at (8,16,4096,4096) and (2,16,16384,4096) against the oracle's `sdpa_heads` (fp32, host);
  * a depth-2 IDDPM training step at 4096 tokens against the oracle's autograd.

The oracle runs on the host cores (a c3 block is ~1.8 TFLOP of fp32: seconds on the GPU box).  Measured values ->
gpurun_out/parity.txt.  These shapes walk every CTA through many tiles (32 KV stages, 14 waves of attention CTAs, 1300+
GEMM tiles), i.e. the phase-wrap / index range the small-geometry tests cannot reach.
"""
import os

import pytest
import torch

from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

if torch.cuda.is_available():
    from pixart_sigma_b200 import PixArtMS, build_model, lib
    from pixart_sigma_b200.training import IDDPMLoss


def _log(line):
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "parity.txt"), "a") as f:
        f.write(line + "\n")


def _rounded(sd):
    return {k: v.to(torch.bfloat16).float() for k, v in sd.items()}


def _one_block_model(sr):
    cfg = po.OracleConfig(depth=1, kv_sampling="conv" if sr > 1 else None, kv_scale_factor=sr,
                          kv_compress_layer=[0] if sr > 1 else [])
    sd = po.synthetic_state_dict(cfg, seed=7)
    kvc = dict(sampling="conv", scale_factor=sr, kv_compress_layer=[0]) if sr > 1 else None
    with torch.device("cuda"):
        m = PixArtMS(depth=1, input_size=32, pe_interpolation=0.5, model_max_length=300, kv_compress_config=kvc)
    m.load_state_dict(sd, strict=False)
    return cfg, _rounded(sd), m.to(torch.bfloat16).eval()


@pytest.mark.parametrize("name,B,hw,lens,sr,fused", [
    ("c3", 8, (64, 64), [300, 8, 77, 300, 129, 128, 255, 64], 1, True),
    ("c3", 8, (64, 64), [300, 8, 77, 300, 129, 128, 255, 64], 1, False),
    ("c4", 2, (128, 128), [300, 41], 2, True),
])
def test_block_at_bench_geometry_matches_oracle(name, B, hw, lens, sr, fused):
    C, N = 1152, hw[0] * hw[1]
    cfg, sdr, m = _one_block_model(sr)
    blk = m.blocks[0]
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, N, C, generator=g)
    t0 = torch.randn(B, 6 * C, generator=g) * 0.3
    ycat = torch.randn(sum(lens), C, generator=g).to(torch.bfloat16)
    mod = (sdr["blocks.0.scale_shift_table"][None] + t0.view(B, 6, C)).cuda().contiguous()
    kv_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
    kv_off = torch.tensor([sum(lens[:i]) for i in range(B)], dtype=torch.int32, device="cuda")
    x32 = x.reshape(B * N, C).cuda().contiguous()
    ln = None
    if fused:        # the model default: LayerNorm + modulate inside the QKV / fc1 GEMM epilogues
        from pixart_sigma_b200.model import _LnFusion, _ln_ctx
        u, v, one_plus = _LnFusion([blk]).prepare(t0.view(B, 6, C).cuda(), mod[None], blk._ws)
        ln = _ln_ctx(u, v, one_plus, 0, torch.empty(B * N, 8, 2, device="cuda"))
    with torch.no_grad():
        got = blk.run_kernels(x32, ycat.cuda(), kv_len, kv_off, max(lens), mod, B, N, hw, blk._ws, ln).view(B, N, C).cpu()
    torch.set_num_threads(min(os.cpu_count() or 1, 64))
    with torch.no_grad():
        want = po.block_forward(sdr, "blocks.0", x, ycat.float()[None], t0, lens, hw, 16, cfg.sr_ratio(0), cfg.kv_sampling)
    err, upd = po.rel_err(got, want), po.rel_err(got - x, want - x)
    per_sample = [po.rel_err(got[b], want[b]) for b in range(B)]
    _log(f"bench-geometry block {name} B={B} hw={hw} lens={lens} sr={sr} fused_ln={fused}: out rel_err={err:.3e} "
         f"update rel_err={upd:.3e} per sample " + " ".join(f"{e:.2e}" for e in per_sample))
    assert torch.isfinite(got).all()
    # the north_star bar on the block output; a sample with very few caption tokens (8 keys: an almost un-averaged, i.e.
    # larger, cross-attention update carrying the same relative bf16 error) sits above the batch figure: 2e-3 per sample
    assert err < (1e-3 if sr == 1 else 1.5e-3), err
    assert max(per_sample) < 2e-3, per_sample


@pytest.mark.parametrize("B,H,Nq,Nk", [(8, 16, 4096, 4096), (2, 16, 16384, 4096)])
@pytest.mark.parametrize("fp32_p", [False, True])
@pytest.mark.parametrize("rev", [False, True])
def test_flash_attn_at_bench_geometry(B, H, Nq, Nk, fp32_p, rev):
    g = torch.Generator().manual_seed(30)
    q = torch.randn(B, Nq, H, 72, generator=g).to(torch.bfloat16)
    k = torch.randn(B, Nk, H, 72, generator=g).to(torch.bfloat16)
    v = torch.randn(B, Nk, H, 72, generator=g).to(torch.bfloat16)
    out = torch.full((B * Nq, H * 72), float("nan"), dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B, H, Nq, dtype=torch.float32, device="cuda")
    st = (H * 72, 72)
    lib.flash_attn(q.cuda(), k.cuda(), v.cuda(), out, B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=B * Nk, q_strides=st, k_strides=st,
                   v_strides=st, lse=lse, fp32_p=fp32_p, reverse_batch=rev)
    got = out.float().cpu().view(B, Nq, H, 72)
    assert torch.isfinite(got).all()
    torch.set_num_threads(min(os.cpu_count() or 1, 64))
    worst = 0.0
    for b in range(B):                                           # the oracle per sample keeps the host working set small
        want = po.sdpa_heads(q[b:b + 1].float(), k[b:b + 1].float(), v[b:b + 1].float())
        worst = max(worst, po.rel_err(got[b:b + 1], want))
        s = torch.einsum("qhd,khd->hqk", q[b, :256].float(), k[b].float()) * (72 ** -0.5)
        want_lse = torch.logsumexp(s, dim=-1) * 1.4426950408889634      # the kernel keeps log2-domain statistics
        assert po.rel_err(lse[b, :, :256].cpu(), want_lse) < 1e-4
    _log(f"bench-geometry flash_attn B={B} H={H} Nq={Nq} Nk={Nk} fp32_p={fp32_p} reverse_batch={rev}: worst per-sample rel_err={worst:.3e}")
    assert worst < 6e-3


def test_train_step_depth2_at_4096_tokens_matches_oracle():
    """IDDPM loss forward + backward of a depth-2 model at the c5 token count (1024px, 4096 tokens, B=2, ragged captions)."""
    from oracle.gen_golden_train import train_inputs
    cfg = po.OracleConfig(depth=2, input_size=128, pe_interpolation=2.0)
    sdr = _rounded(po.synthetic_state_dict(cfg, seed=0))
    x0, t, y, mask, noise = train_inputs(cfg, 2, (128, 128), [17, 803], [300, 50])
    r = lambda v_: v_.to(torch.bfloat16).float()
    kw = dict(type="PixArtMS", depth=2, input_size=128, pe_interpolation=2.0, model_max_length=300)
    with torch.device("cuda"):
        m = build_model(kw)
    m.load_state_dict(sdr, strict=False)
    m = m.float().train()
    m.y_embedder.uncond_prob = 0.0
    loss = IDDPMLoss()
    terms = loss.training_losses(m, x0.cuda(), t.cuda(), dict(y=r(y).cuda(), mask=mask.cuda(), data_info=None), noise=noise.cuda())
    terms["loss"].mean().backward()
    torch.set_num_threads(min(os.cpu_count() or 1, 64))
    sdo = {k_: v_.clone().requires_grad_(v_.is_floating_point()) for k_, v_ in sdr.items()}
    ref = loss.training_losses(lambda xx, timestep, **k_: po.forward_grad(sdo, cfg, xx, timestep.float(), k_["y"], mask=k_["mask"]),
                               x0, t, dict(y=r(y), mask=mask, data_info=None), noise=noise)
    ref["loss"].mean().backward()
    lt = max(po.rel_err(terms[k_].detach().cpu(), ref[k_].detach()) for k_ in ("mse", "vb", "loss"))
    errs = {n: po.rel_err(p.grad.float().cpu(), sdo[n].grad) for n, p in m.named_parameters()}
    worst = max(errs, key=errs.get)
    _log(f"bench-geometry train step depth 2, 4096 tokens, B=2: loss vs oracle {lt:.2e}; grads max {errs[worst]:.2e} ({worst})")
    assert lt < 2e-3
    assert errs[worst] < 2e-2, (worst, errs[worst])
