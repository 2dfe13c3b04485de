"""Blocks on token grids whose sides are odd or not multiples of the KV scale factor (-m gpu), against the oracle block:
B = 3 samples of N = 255 (15 x 17) or 243 (9 x 27) tokens put the sample boundaries inside the 16-row warp blocks of
ln_modulate_bwd and the 32-row CTAs of gate_residual_bwd; 15 x 17 and 9 x 27 are token grids of non-square aspect buckets.

The parameter-free KV samplings are checked where the reference's rule and the [::sr, ::sr] pick part ways: 'ave' is
nearest-neighbour interpolation by 1/sr (PixArt_blocks.py:109-112), which keeps floor(H/sr) x floor(W/sr) keys.
'uniform_every' runs at sr = 3, which divides both token counts (the reference rejects sr = 2 on an odd token count;
tests/test_kv_pick_cpu.py checks that the native paths do too).  Captions of 300, 77 and 120 tokens.

Bounds as in test_training_gpu.py (training forward 2e-3, every gradient 2e-2 normwise; the checkpointed block agrees with
the plain one) and test_model_gpu.py (inference block 1e-3)."""
import pytest
import torch

from oracle import pixart_oracle as po
from test_model_gpu import _bf16_round, _build
from test_training_gpu import _assert_checkpointing_agrees, _kernel_block_grads, _log, _rounded

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import build_model

B, C, LENS = 3, 1152, [300, 77, 120]
TRAIN_CASES = [(None, 1, (15, 17)), (None, 1, (9, 27)), ("ave", 2, (15, 17)), ("ave", 2, (9, 27)), ("ave", 3, (16, 16)),
               ("uniform_every", 3, (15, 17)), ("uniform_every", 3, (9, 27))]


def _cfg(sampling, sr):
    return po.OracleConfig(depth=1, kv_sampling=sampling, kv_scale_factor=sr, kv_compress_layer=[0] if sampling else [])


def _d64(t):
    """The oracle runs in float64 on the GPU: a stricter reference than fp32 on the CPU, and fast at B = 3."""
    return t.double().cuda()


def _inputs(hw, seed):
    g = torch.Generator().manual_seed(seed)
    N = hw[0] * hw[1]
    x = torch.randn(B, N, C, generator=g)
    t0 = torch.randn(B, 6 * C, generator=g) * 0.3
    ycat = torch.randn(sum(LENS), C, generator=g).to(torch.bfloat16).float()
    dout = torch.randn(B, N, C, generator=g)
    return x, t0, ycat, dout


@pytest.mark.parametrize("sampling,sr,hw", TRAIN_CASES)
def test_block_gradients_on_odd_token_grids_match_oracle(sampling, sr, hw):
    """BlockFn forward + backward on the kernels vs the oracle block's float64 autograd on the same bf16-rounded weights, then
    the activation-checkpointed block against the plain one."""
    cfg = _cfg(sampling, sr)
    sd = _rounded(po.synthetic_state_dict(cfg, seed=7))
    kw = dict(type="PixArtMS", depth=1, input_size=32, pe_interpolation=0.5, model_max_length=300)
    if sampling:
        kw["kv_compress_config"] = dict(sampling=sampling, scale_factor=sr, kv_compress_layer=[0])
    with torch.device("cuda"):
        m = build_model(kw)
    m.load_state_dict(sd, strict=False)
    blk = m.float().train().blocks[0]
    x, t0, ycat, dout = _inputs(hw, seed=11)
    sdo = {k: _d64(v).requires_grad_(True) for k, v in sd.items() if k.startswith("blocks.0.")}
    xo = _d64(x).requires_grad_(True)
    want = po.block_forward(sdo, "blocks.0", xo, _d64(ycat)[None], _d64(t0), LENS, hw, 16, sr, sampling)
    want.backward(_d64(dout))
    got, grads = _kernel_block_grads(blk, x, ycat, t0, dout, LENS, hw, False)
    ferr = po.rel_err(got, want.detach().cpu())
    errs = {"x": po.rel_err(grads["x"], xo.grad.cpu())}
    for n, _ in blk.named_parameters():
        errs[n] = po.rel_err(grads[n], sdo["blocks.0." + n].grad.cpu())
    worst = max(errs, key=errs.get)
    line = f"block grads {sampling} sr={sr} hw={hw} B={B}: fwd={ferr:.2e} max grad err {errs[worst]:.2e} ({worst})"
    print(line)
    _log(line)
    assert ferr < 2e-3, ferr
    assert errs[worst] < 2e-2, errs
    _assert_checkpointing_agrees(blk, x, ycat, t0, dout, LENS, hw, grads)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("sr,hw", [(2, (15, 17)), (2, (9, 27)), (3, (16, 16))])
def test_ave_block_forward_on_odd_token_grids_matches_oracle_1e3(sr, hw, fused):
    """The inference block (run_kernels, fp32 residual stream) with 'ave' KV sampling vs the oracle block: the 1e-3 bar of
    test_block_forward_matches_oracle_1e3.  The picked keys are bf16 rows of the QKV output, as without compression."""
    N = hw[0] * hw[1]
    cfg = _cfg("ave", sr)
    sd = po.synthetic_state_dict(cfg, seed=7)
    m = _build(cfg, sd)
    blk = m.blocks[0]
    x, t0, ycat, _ = _inputs(hw, seed=11)
    ycat = ycat.to(torch.bfloat16)
    sdr = _bf16_round(sd)
    want = po.block_forward({k: _d64(v) for k, v in sdr.items()}, "blocks.0", _d64(x), _d64(ycat)[None], _d64(t0), LENS, hw, 16,
                            sr, "ave").cpu()
    mod = (sdr["blocks.0.scale_shift_table"][None] + t0.view(B, 6, C)).cuda().contiguous()
    kv_len = torch.tensor(LENS, dtype=torch.int32, device="cuda")
    kv_off = torch.tensor([sum(LENS[:i]) for i in range(B)], dtype=torch.int32, device="cuda")
    x32 = x.reshape(B * N, C).cuda().contiguous()
    ln = None
    if fused:
        from pixart_sigma_b200.model import _LnFusion, _ln_ctx
        u, v, one_plus = _LnFusion([blk]).prepare(t0.view(B, 6, C).cuda(), mod[None], blk._ws)
        ln = _ln_ctx(u, v, one_plus, 0, torch.empty(B * N, 8, 2, device="cuda"))
    with torch.no_grad():
        got = blk.run_kernels(x32, ycat.cuda(), kv_len, kv_off, max(LENS), mod, B, N, hw, blk._ws, ln).view(B, N, C).cpu()
    err = po.rel_err(got, want)
    line = f"ave block forward sr={sr} hw={hw} fused_ln={fused}: out rel_err={err:.3e} update rel_err={po.rel_err(got - x, want - x):.3e}"
    print(line)
    _log(line)
    assert err < 1e-3, err
