"""GPU parity tests (-m gpu) of the training path (forward + backward kernels under torch autograd):
 (a) PixArtMSBlock gradients vs the oracle block's autograd in fp32 on the same bf16-rounded weights / inputs;
 (b) a depth-2 model's IDDPM training step vs the oracle (same rounding) and vs the gradient fingerprints of the
     UNMODIFIED reference (tests/golden/train_*.pt, fp32 weights -> adds the bf16 weight-rounding floor);
 (c) activation checkpointing (set_grad_checkpoint attrs) and bf16 parameters give the same gradients.

Tolerances (normwise rel-err per gradient tensor): every matmul operand on the backward path is bf16 (activations,
P / dS of the attention, the gradients flowing between ops), so a gradient tensor carries a few bf16 roundings per
layer it passes: 2e-2 vs (a), 3e-2 vs the reference fixtures.  Loss terms: 2e-3.  Measured values -> gpurun_out/parity.txt.
"""
import os

import pytest
import torch

from oracle import pixart_oracle as po
from oracle.gen_golden_train import fingerprint_positions, train_inputs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

if torch.cuda.is_available():
    from pixart_sigma_b200 import PixArtMS, build_model
    from pixart_sigma_b200.parallel import GradBucketReducer
    from pixart_sigma_b200.training import GraphedTrainStep, IDDPMLoss, train_step


def _log(line):
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "parity.txt"), "a") as f:
        f.write(line + "\n")


def _rounded(sd):
    return {k: v.to(torch.bfloat16).float() for k, v in sd.items()}


def _build_train(cfg, sd, dtype=torch.float32, checkpoint=False):
    kw = dict(type="PixArtMS", depth=cfg.depth, hidden_size=cfg.hidden_size, num_heads=cfg.num_heads,
              input_size=cfg.input_size, pe_interpolation=cfg.pe_interpolation, model_max_length=cfg.model_max_length)
    if cfg.kv_sampling is not None:
        kw["kv_compress_config"] = dict(sampling=cfg.kv_sampling, scale_factor=cfg.kv_scale_factor,
                                        kv_compress_layer=list(cfg.kv_compress_layer))
    with torch.device("cuda"):
        m = build_model(kw, use_grad_checkpoint=checkpoint)
    m.load_state_dict(sd, strict=False)
    m = m.to(dtype).train()
    m.y_embedder.uncond_prob = 0.0            # caption dropout is random; the fixtures were made without it
    return m


@pytest.mark.parametrize("B,hw,lens", [(2, (16, 16), [300, 77]), (1, (16, 24), [120])])
def test_block_gradients_match_oracle(B, hw, lens):
    C, N = 1152, hw[0] * hw[1]
    cfg = po.OracleConfig(depth=1)
    sd = _rounded(po.synthetic_state_dict(cfg, seed=7))
    m = _build_train(cfg, sd)
    blk = m.blocks[0]
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, N, C, generator=g)
    t0 = torch.randn(B, 6 * C, generator=g) * 0.3
    ycat = torch.randn(sum(lens), C, generator=g).to(torch.bfloat16).float()
    dout = torch.randn(B, N, C, generator=g)
    # oracle autograd
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k.startswith("blocks.0.")}
    xo, to, yo = x.clone().requires_grad_(True), t0.clone().requires_grad_(True), ycat.clone().requires_grad_(True)
    want = po.block_forward(sdo, "blocks.0", xo, yo[None], to, lens, hw, 16, 1, None)
    want.backward(dout)
    # kernels, through the reference block signature (fp32 in/out here so that the comparison sees only kernel error)
    xk, tk, yk = (v.clone().cuda().requires_grad_(True) for v in (x, t0, ycat))
    got = blk(xk, yk[None], tk, lens, hw)
    # the training forward keeps each branch output in bf16 before the (fp32) gated residual add -- one rounding more
    # than the fused inference epilogue, which is held to 1e-3 (test_model_gpu.py)
    ferr = po.rel_err(got.detach().cpu(), want.detach())
    assert ferr < 1.5e-3, ferr
    got.backward(dout.cuda())
    errs = {"x": po.rel_err(xk.grad.cpu(), xo.grad), "t": po.rel_err(tk.grad.cpu(), to.grad),
            "y": po.rel_err(yk.grad.cpu(), yo.grad)}
    for n, p in blk.named_parameters():
        errs[n] = po.rel_err(p.grad.float().cpu(), sdo["blocks.0." + n].grad)
    _log(f"block grads B={B} hw={hw} lens={lens}: " + " ".join(f"{k}={v:.2e}" for k, v in errs.items()))
    assert max(errs.values()) < 2e-2, errs


def _kernel_block_grads(blk, x, ycat, t0, dout, lens, hw, ckpt):
    """(output, {"x": x.grad, parameter name: .grad}) of one kernel block forward + backward, activation-checkpointed or not."""
    blk.grad_checkpointing = ckpt
    blk.zero_grad(set_to_none=True)
    xk = x.clone().cuda().requires_grad_(True)
    got = blk(xk, ycat.cuda()[None], t0.cuda(), lens, hw)
    got.backward(dout.cuda())
    return got.detach().cpu(), {"x": xk.grad.cpu(), **{n: p.grad.float().cpu() for n, p in blk.named_parameters()}}


def _assert_checkpointing_agrees(blk, x, ycat, t0, dout, lens, hw, grads):
    """The checkpointed block gives the gradients `grads` of the plain one (atomics reorder sums)."""
    _, ck = _kernel_block_grads(blk, x, ycat, t0, dout, lens, hw, True)
    for n in grads:
        assert torch.equal(ck[n], grads[n]) or po.rel_err(ck[n], grads[n]) < 1e-5, (n, po.rel_err(ck[n], grads[n]))


@pytest.mark.parametrize("sampling", ["conv", "uniform", "uniform_every"])
def test_kv_compressed_block_gradients_match_oracle(sampling):
    """Training through a KV-compressed block (PixArt_blocks.py:97-121, 137-139): conv + LN compression kernel and its
    backward, attention backward with Nk = N / 4 (N / 2 for uniform_every); then the activation-checkpointed block against
    the plain one."""
    B, hw, lens, C = 2, (16, 16), [300, 9], 1152
    N = hw[0] * hw[1]
    cfg = po.OracleConfig(depth=1, kv_sampling=sampling, kv_scale_factor=2, kv_compress_layer=[0])
    sd = _rounded(po.synthetic_state_dict(cfg, seed=7))
    kw = dict(type="PixArtMS", depth=1, input_size=32, pe_interpolation=0.5, model_max_length=300,
              kv_compress_config=dict(sampling=sampling, scale_factor=2, kv_compress_layer=[0]))
    with torch.device("cuda"):
        m = build_model(kw)
    m.load_state_dict(sd, strict=False)
    blk = m.float().train().blocks[0]
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, N, C, generator=g)
    t0 = torch.randn(B, 6 * C, generator=g) * 0.3
    ycat = torch.randn(sum(lens), C, generator=g).to(torch.bfloat16).float()
    dout = torch.randn(B, N, C, generator=g)
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k.startswith("blocks.0.")}
    xo = x.clone().requires_grad_(True)
    want = po.block_forward(sdo, "blocks.0", xo, ycat[None], t0, lens, hw, 16, 2, sampling)
    want.backward(dout)
    got, grads = _kernel_block_grads(blk, x, ycat, t0, dout, lens, hw, False)
    ferr = po.rel_err(got, want.detach())
    assert ferr < 2e-3, ferr
    errs = {"x": po.rel_err(grads["x"], xo.grad)}
    for n, _ in blk.named_parameters():
        errs[n] = po.rel_err(grads[n], sdo["blocks.0." + n].grad)
    _log(f"kv-compressed ({sampling}) block grads: fwd={ferr:.2e} " + " ".join(f"{k}={v:.2e}" for k, v in errs.items()))
    assert max(errs.values()) < 2e-2, errs
    _assert_checkpointing_agrees(blk, x, ycat, t0, dout, lens, hw, grads)


def test_qk_norm_block_gradients_match_oracle():
    """Training with qk_norm=True (PixArt_blocks.py:133-134): q_norm / k_norm on the qkv GEMM output, their backward through the
    LayerNorm-modulate backward kernel, inside autograd.BlockFn; then the activation-checkpointed block against the plain
    one."""
    B, hw, lens, C = 2, (16, 16), [300, 40], 1152
    N = hw[0] * hw[1]
    cfg = po.OracleConfig(depth=1, qk_norm=True)
    sd = _rounded(po.synthetic_state_dict(cfg, seed=9))
    kw = dict(type="PixArtMS", depth=1, input_size=32, pe_interpolation=0.5, model_max_length=300, qk_norm=True)
    with torch.device("cuda"):
        m = build_model(kw)
    m.load_state_dict(sd, strict=False)
    blk = m.float().train().blocks[0]
    g = torch.Generator().manual_seed(13)
    x = torch.randn(B, N, C, generator=g)
    t0 = torch.randn(B, 6 * C, generator=g) * 0.3
    ycat = torch.randn(sum(lens), C, generator=g).to(torch.bfloat16).float()
    dout = torch.randn(B, N, C, generator=g)
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k.startswith("blocks.0.")}
    xo = x.clone().requires_grad_(True)
    want = po.block_forward(sdo, "blocks.0", xo, ycat[None], t0, lens, hw, 16, 1, None, True)
    want.backward(dout)
    got, grads = _kernel_block_grads(blk, x, ycat, t0, dout, lens, hw, False)
    ferr = po.rel_err(got, want.detach())
    assert ferr < 2e-3, ferr
    errs = {"x": po.rel_err(grads["x"], xo.grad)}
    for n, _ in blk.named_parameters():
        if n == "attn.k_norm.bias":
            # a constant added to every key moves all logits of a query by the same amount: the exact gradient is ZERO and both
            # sides hold rounding noise only -- compare its size with the (real) gradient of q_norm.bias instead
            errs[n] = (grads[n].norm() / grads["attn.q_norm.bias"].norm()).item()
            continue
        errs[n] = po.rel_err(grads[n], sdo["blocks.0." + n].grad)
    _log(f"qk_norm block grads: fwd={ferr:.2e} " + " ".join(f"{k}={v:.2e}" for k, v in errs.items()))
    assert max(errs.values()) < 2e-2, errs
    _assert_checkpointing_agrees(blk, x, ycat, t0, dout, lens, hw, grads)


def _oracle_step(cfg, sd, x0, t, y, mask, noise):
    sdo = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    model = lambda x, timestep, **kw: po.forward_grad(sdo, cfg, x, timestep.float(), kw["y"], mask=kw["mask"])
    terms = IDDPMLoss().training_losses(model, x0, t, dict(y=y, mask=mask, data_info=None), noise=noise)
    terms["loss"].mean().backward()
    return {k: v.detach() for k, v in terms.items()}, {k: v.grad for k, v in sdo.items() if v.grad is not None}


@pytest.mark.parametrize("name", ["train_d2_b2", "train_d2_b3_512", "train_d2_kvconv"])
def test_train_step_matches_oracle_and_reference_fixture(golden_dir, name):
    fix = torch.load(os.path.join(golden_dir, name + ".pt"))
    cfg = po.OracleConfig(**fix["cfg"])
    sd = po.synthetic_state_dict(cfg, seed=0)
    x0, t, y, mask, noise = train_inputs(cfg, fix["batch"], tuple(fix["hw"]), fix["t"], fix["lens"])
    r = lambda v: v.to(torch.bfloat16).float()
    sdr = _rounded(sd)
    m = _build_train(cfg, sdr)
    loss = IDDPMLoss()
    terms = loss.training_losses(m, x0.cuda(), t.cuda(), dict(y=r(y).cuda(), mask=mask.cuda(), data_info=None), noise=noise.cuda())
    terms["loss"].mean().backward()
    want_terms, want = _oracle_step(cfg, sdr, x0, t, r(y), mask, noise)
    e_or, e_fix = {}, {}
    for n, p in m.named_parameters():
        g = p.grad.float().cpu()
        e_or[n] = po.rel_err(g, want[n])
        ref = fix["grads"][n]
        e_fix[n] = max(po.rel_err(g.flatten()[fingerprint_positions(g.numel())], ref["vals"]),
                       abs(float(g.norm()) - float(ref["norm"])) / float(ref["norm"]))
    lt = max(po.rel_err(terms[k].cpu(), want_terms[k]) for k in ("mse", "vb", "loss"))
    lf = max(po.rel_err(terms[k].cpu(), fix["terms"][k]) for k in ("mse", "vb", "loss"))
    wo, wf = max(e_or, key=e_or.get), max(e_fix, key=e_fix.get)
    _log(f"train {name}: loss vs oracle {lt:.2e} vs reference {lf:.2e}; grads vs oracle max {e_or[wo]:.2e} ({wo}), "
         f"vs reference fixture max {e_fix[wf]:.2e} ({wf})")
    assert lt < 2e-3 and lf < 5e-3
    assert e_or[wo] < 2e-2, (wo, e_or[wo])
    assert e_fix[wf] < 3e-2, (wf, e_fix[wf])


def test_checkpointing_and_bf16_parameters_give_the_same_gradients():
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    sd = _rounded(po.synthetic_state_dict(cfg, seed=0))
    x0, t, y, mask, noise = train_inputs(cfg, 2, (32, 32), [10, 600], [300, 50])
    args = (x0.cuda(), t.cuda(), y.cuda(), mask.cuda())
    grads = []
    for dtype, ckpt in ((torch.float32, False), (torch.float32, True), (torch.bfloat16, True)):
        m = _build_train(cfg, sd, dtype=dtype, checkpoint=ckpt)
        if ckpt:
            assert all(getattr(b, "grad_checkpointing", False) for b in m.blocks)
        m.output_dtype = torch.float32
        lval = train_step(m, IDDPMLoss(), *args, noise=noise.cuda())
        assert torch.isfinite(lval)
        grads.append({n: p.grad.float().clone() for n, p in m.named_parameters()})
    for n in grads[0]:
        assert torch.equal(grads[0][n], grads[1][n]) or po.rel_err(grads[1][n], grads[0][n]) < 1e-5, n   # atomics reorder sums
        assert po.rel_err(grads[2][n], grads[0][n]) < 2e-2, n                                          # bf16 grads / params


@pytest.mark.parametrize("ckpt", [False, True])
def test_graphed_train_step_equals_eager_and_sees_parameter_updates(ckpt):
    """The whole step (zero-grad + loss fwd + bwd, with or without activation checkpointing) replayed from one CUDA
    graph gives the eager gradients, also after the parameters were updated in place between replays."""
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    sd = _rounded(po.synthetic_state_dict(cfg, seed=0))
    x0, t, y, mask, noise = train_inputs(cfg, 2, (32, 32), [10, 600], [300, 50])
    batch = tuple(v.cuda() for v in (x0, t, y.to(torch.bfloat16), mask, noise))
    m = _build_train(cfg, sd, checkpoint=ckpt)
    red = GradBucketReducer(m)
    loss = IDDPMLoss()

    def eager():
        red.zero_grad()
        lv = train_step(m, loss, batch[0], batch[1], batch[2], batch[3], noise=batch[4], reducer=red)
        return lv.clone(), {n: p.grad.clone() for n, p in m.named_parameters()}

    l0, g0 = eager()
    step = GraphedTrainStep(m, loss, red, batch)
    lg = step(*batch).clone()
    assert po.rel_err(lg, l0) < 1e-5
    for n, p in m.named_parameters():
        assert po.rel_err(p.grad, g0[n]) < 1e-4, n              # atomics reorder fp32 sums
    with torch.no_grad():                                       # an "optimizer step"
        for p in m.parameters():
            p.add_(0.01 * torch.randn_like(p))
    lg2 = step(*batch).clone()
    g2 = {n: p.grad.clone() for n, p in m.named_parameters()}
    l1, g1 = eager()
    assert abs(float(l1) - float(l0)) > 1e-6                    # the update changed the loss ...
    assert po.rel_err(lg2, l1) < 1e-5                           # ... and the replay saw it (shadows refreshed in place)
    for n in g1:
        assert po.rel_err(g2[n], g1[n]) < 1e-4, n


def test_flat_adamw_matches_torch_adamw():
    """`optim.FlatAdamW` (one pxa_adamw_flat launch per gradient bucket, parameters flattened in place) against
    torch.optim.AdamW with the reference's hyper-parameters (configs/PixArt_xl2_internal.py:48), three steps."""
    from pixart_sigma_b200.optim import FlatAdamW

    class Tiny(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.blocks = torch.nn.ModuleList([torch.nn.Linear(37, 53) for _ in range(2)])
            self.head = torch.nn.Linear(53, 7)

    torch.manual_seed(0)
    a, b = Tiny().cuda(), Tiny().cuda()
    b.load_state_dict(a.state_dict())
    red = GradBucketReducer(a)
    opt = FlatAdamW(red, lr=2e-3, eps=1e-10, weight_decay=3e-2)
    ref = torch.optim.AdamW(b.parameters(), lr=2e-3, eps=1e-10, weight_decay=3e-2)
    for (_, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.equal(pa, pb)                                # flattening kept the values
    g = torch.Generator(device="cuda").manual_seed(1)
    for step in range(3):
        for pa, pb in zip(a.parameters(), b.parameters()):
            gr = torch.randn(pa.shape, device="cuda", generator=g)
            pa.grad.copy_(gr)                                     # the bucket view
            pb.grad = gr.clone()
        opt.step()
        ref.step()
        for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
            assert po.rel_err(pa, pb) < 1e-6, (step, n)
    sd = opt.state_dict()
    assert sd["step"] == 3 and len(sd["state"]) == len(red.buckets)


def test_direct_gradient_accumulation_equals_autograd_accumulation():
    """With a GradBucketReducer the weight / bias gradient kernels accumulate straight into the bucket views (no autograd
    accumulation pass); the result must equal the gradients autograd accumulates without a reducer, also over two
    accumulation steps, and the reducer must have seen every bucket complete."""
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    sd = _rounded(po.synthetic_state_dict(cfg, seed=0))
    x0, t, y, mask, noise = train_inputs(cfg, 2, (32, 32), [10, 600], [300, 50])
    args = (x0.cuda(), t.cuda(), y.cuda(), mask.cuda())
    plain = _build_train(cfg, sd, checkpoint=True)
    for _ in range(2):
        train_step(plain, IDDPMLoss(), *args, noise=noise.cuda())
    direct = _build_train(cfg, sd, checkpoint=True)
    red = GradBucketReducer(direct)
    red.zero_grad()
    for _ in range(2):
        train_step(direct, IDDPMLoss(), *args, noise=noise.cuda(), reducer=red)
        assert all(b["pending"] == 0 for b in red.buckets), {b["key"]: b["pending"] for b in red.buckets}   # all reported
    for (n, pa), (_, pb) in zip(plain.named_parameters(), direct.named_parameters()):
        assert po.rel_err(pb.grad, pa.grad) < 1e-4, n
