"""LoRA fine-tuning on the kernels (-m gpu): the adapter-aware training forward / backward (GEMM K-tail, skinny down- and
up-projections, adapter-only weight gradients) against the oracle's peft LoRA layers (oracle/lora_oracle.py) in fp32 on the
same bf16-rounded weights, optimizer steps against torch's AdamW, the adapter file round trip, graph capture and the absence of
host syncs.  Bounds are normwise per tensor, as in test_training_gpu.py: loss 2e-3, gradients 2e-2.  The measured values are
printed (pytest -s shows them)."""
import pytest
import torch

from oracle import lora_oracle as lo
from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import build_model, lora
    from pixart_sigma_b200.optim import FlatAdamW, clip_grad_norm_
    from pixart_sigma_b200.parallel import GradBucketReducer
    from pixart_sigma_b200.training import DDPMEpsLoss, GraphedTrainStep, train_step

KINDS = {"plain": ({}, {}),
         "kv_compress": (dict(kv_sampling="conv", kv_scale_factor=2, kv_compress_layer=[0]),
                         dict(kv_compress_config=dict(sampling="conv", scale_factor=2, kv_compress_layer=[0]))),
         "qk_norm": (dict(qk_norm=True), dict(qk_norm=True))}
R = 4                      # rank 4: s = 8 / 4 = 2 (exact); T = 8 (padded from 4), 16 (qkv, from 12), 8 (kv)


def _log(line):
    print(line)


def _r(v):
    return v.to(torch.bfloat16).float()


def _setup(kind="plain", ckpt=False, zero_b=False, seed=0):
    """A depth-2 fp32 model on bf16-rounded weights with a rank-4 adapter (bf16-representable A and, unless zero_b, B)."""
    ckw, mkw = KINDS[kind]
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5, **ckw)
    sd = {k: _r(v) for k, v in po.synthetic_state_dict(cfg, seed=3).items()}
    kw = dict(type="PixArtMS", depth=2, input_size=32, pe_interpolation=0.5, model_max_length=300, class_dropout_prob=0.0, **mkw)
    with torch.device("cuda"):
        m = build_model(kw, use_grad_checkpoint=ckpt)
    m.load_state_dict(sd, strict=False)
    m = m.float().train()
    lora.inject_lora(m, R, generator=torch.Generator().manual_seed(seed))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for _, mod in lora._adapted(m):
            mod.lora_A.copy_(_r(mod.lora_A))
            if not zero_b:
                mod.lora_B.copy_(_r(torch.randn(mod.lora_B.shape, generator=g) * 0.02))
    return cfg, sd, m


def _inputs(cfg):
    x, _, y, mask = po.synthetic_inputs(cfg, 2, (32, 32), lens=[300, 77])
    g = torch.Generator().manual_seed(5)
    return x * 0.5, torch.tensor([17, 803]), _r(y), mask, torch.randn(x.shape, generator=g)


def _native_loss(m, loss, x0, t, y, mask, noise):
    kw = dict(y=y.cuda(), mask=mask.cuda(), data_info=None)
    return loss.training_losses(m, x0.cuda(), t.cuda(), kw, noise=noise.cuda())["loss"].mean()


def _oracle_adapters(m):
    return {n: (mod.lora_A.detach().float().cpu().clone().requires_grad_(),
                mod.lora_B.detach().float().cpu().clone().requires_grad_()) for n, mod in lora._adapted(m)}


def _oracle_loss(sd, ad, cfg, x0, t, y, mask, noise):
    fn = lambda xx, timestep, **kw: lo.forward_grad(sd, ad, 2.0, cfg, xx, timestep.float(), kw["y"], mask=kw["mask"])
    return DDPMEpsLoss().training_losses(fn, x0, t, dict(y=y, mask=mask), noise=noise)["loss"].mean()


def test_fresh_adapter_is_bitwise_the_base_forward_and_trains_only_the_adapter():
    cfg, sd, m = _setup(zero_b=True)
    x0, t, y, mask, noise = _inputs(cfg)
    # the same model without the adapter, on the same weights
    with torch.device("cuda"):
        ref = build_model(dict(type="PixArtMS", depth=2, input_size=32, pe_interpolation=0.5, model_max_length=300,
                               class_dropout_prob=0.0))
    ref.load_state_dict(m.state_dict(), strict=False)
    ref = ref.float().train()
    kw = dict(y=y.cuda(), mask=mask.cuda(), data_info=None)
    want = ref(x0.cuda(), t.cuda(), **kw)
    red = GradBucketReducer(m)
    got = m(x0.cuda(), t.cuda(), **kw)
    assert got.requires_grad and torch.equal(got.detach(), want.detach())
    got.square().mean().backward()
    red.finish()
    names = {id(p): n for n, p in m.named_parameters()}
    assert all(names[id(p)].endswith((".lora_A", ".lora_B")) for b in red.buckets for p in b["params"])
    assert {names[id(p)] for b in red.buckets for p in b["params"]} == {n for n, p in m.named_parameters() if p.requires_grad}
    assert all(p.grad is None for n, p in m.named_parameters() if not n.endswith((".lora_A", ".lora_B")))
    assert any(p.grad.abs().sum() > 0 for n, p in m.named_parameters() if n.endswith(".lora_B"))


@pytest.mark.parametrize("kind", list(KINDS))
def test_adapter_gradients_match_oracle(kind):
    """Every adapter's gradient (qkv / kv groups, the patch-embedding conv, caption projection, t_block, t_embedder, final
    layer) against the oracle's autograd; checkpointing on and off agree to 1e-4."""
    grads = {}
    for ckpt in (False, True):
        cfg, sd, m = _setup(kind, ckpt=ckpt)
        x0, t, y, mask, noise = _inputs(cfg)
        loss = _native_loss(m, DDPMEpsLoss(), x0, t, y, mask, noise)
        loss.backward()
        grads[ckpt] = {n + "." + k: getattr(mod, k).grad.float().cpu() for n, mod in lora._adapted(m) for k in ("lora_A", "lora_B")}
    ad = _oracle_adapters(m)
    want = _oracle_loss(sd, ad, cfg, x0, t, y, mask, noise)
    want.backward()
    lerr = po.rel_err(loss.detach().cpu().reshape(1), want.detach().reshape(1))
    errs = {}
    for n, (A, B) in ad.items():
        errs[n + ".lora_A"] = po.rel_err(grads[False][n + ".lora_A"], A.grad)
        errs[n + ".lora_B"] = po.rel_err(grads[False][n + ".lora_B"], B.grad)
    ck = max(po.rel_err(grads[True][k], grads[False][k]) for k in grads[False])
    worst = max(errs, key=errs.get)
    _log(f"lora grads {kind}: loss {lerr:.2e}, max grad {errs[worst]:.2e} ({worst}), ckpt on/off {ck:.2e}")
    for must in ("x_embedder.proj", "y_embedder.y_proj.fc1", "t_block.1", "t_embedder.mlp.0", "final_layer.linear",
                 "blocks.0.attn.qkv", "blocks.1.cross_attn.kv_linear", "blocks.1.mlp.fc2"):
        assert must + ".lora_A" in errs
    assert lerr < 2e-3 and errs[worst] < 2e-2, errs
    assert ck < 1e-4


def _steps(m, red, opt, x0, t, y, mask, noise, n=3):
    loss = DDPMEpsLoss()
    for _ in range(n):
        red.zero_grad()
        train_step(m, loss, x0.cuda(), t.cuda(), y.cuda(), mask.cuda(), noise=noise.cuda(), reducer=red)
        clip_grad_norm_(red, 1.0)
        opt.step()


def test_three_optimizer_steps_match_torch_adamw():
    cfg, sd, m = _setup()
    x0, t, y, mask, noise = _inputs(cfg)
    ad = _oracle_adapters(m)
    p0 = {n: (A.detach().clone(), B.detach().clone()) for n, (A, B) in ad.items()}
    red = GradBucketReducer(m)
    opt = FlatAdamW(red, lr=1e-5, weight_decay=1e-2, eps=1e-8)
    _steps(m, red, opt, x0, t, y, mask, noise)
    params = [p for pair in ad.values() for p in pair]
    topt = torch.optim.AdamW(params, lr=1e-5, weight_decay=1e-2, eps=1e-8)
    for _ in range(3):
        topt.zero_grad()
        _oracle_loss(sd, ad, cfg, x0, t, y, mask, noise).backward()
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        topt.step()
    got = torch.cat([torch.cat([(mod.lora_A.detach().cpu() - p0[n][0]).flatten(), (mod.lora_B.detach().cpu() - p0[n][1]).flatten()])
                     for n, mod in lora._adapted(m)])
    want = torch.cat([torch.cat([(ad[n][0].detach() - p0[n][0]).flatten(), (ad[n][1].detach() - p0[n][1]).flatten()])
                      for n, _ in lora._adapted(m)])
    err = po.rel_err(got, want)
    _log(f"lora 3 AdamW steps: update rel_err {err:.2e}")
    # Adam divides each gradient element by its own magnitude, so the elements whose gradient lies within the gradients'
    # ~1-2 % bf16 error of zero can take an update of either sign: the normwise update error is several times the
    # gradients' (measured 7.7e-2 on an H100 with these seeds); a wrong gradient moves it to O(1)
    assert err < 1e-1, err


def test_adapter_round_trip_after_training(tmp_path):
    """save_adapter -> fresh model -> load_adapter -> merge_lora: its no-grad forward matches the trained model's unmerged
    training forward (1e-2, test_lora_gpu.py's merged-forward bound); the trained adapter moves the output by more than 10x."""
    cfg, sd, m = _setup(zero_b=True)
    x0, t, y, mask, noise = _inputs(cfg)
    red = GradBucketReducer(m)
    opt = FlatAdamW(red, lr=2e-3, weight_decay=1e-2, eps=1e-8)
    _steps(m, red, opt, x0, t, y, mask, noise, n=3)
    kw = dict(y=y.cuda(), mask=mask.cuda(), data_info=None)
    trained = m(x0.cuda(), t.cuda(), **kw).detach().float().cpu()
    lora.save_adapter(m, str(tmp_path))
    with torch.device("cuda"):
        f = build_model(dict(type="PixArtMS", depth=2, input_size=32, pe_interpolation=0.5, model_max_length=300))
    f.load_state_dict(sd, strict=False)
    with torch.no_grad():
        base = f.to(torch.bfloat16).eval()(x0.cuda(), t.cuda(), **kw).float().cpu()
    f = f.float()
    lora.load_adapter(f, str(tmp_path))
    lora.merge_lora(f)
    f = f.to(torch.bfloat16).eval()
    with torch.no_grad():
        merged = f(x0.cuda(), t.cuda(), **kw).float().cpu()
    err, moved = po.rel_err(merged, trained), po.rel_err(base, trained)
    _log(f"lora round trip: merged vs trained {err:.2e}, adapter moves the output by {moved:.2e}")
    assert err < 1e-2 and moved > 10 * err, (err, moved)


def test_graphed_lora_step_matches_eager_and_sees_updates():
    cfg, sd, m = _setup()
    x0, t, y, mask, noise = _inputs(cfg)
    red = GradBucketReducer(m)
    opt = FlatAdamW(red, lr=1e-4, weight_decay=1e-2, eps=1e-8)
    red.zero_grad()
    eager = train_step(m, DDPMEpsLoss(), x0.cuda(), t.cuda(), y.cuda(), mask.cuda(), noise=noise.cuda(), reducer=red)
    eager_g = torch.cat([b["flat"].clone() for b in red.buckets])
    batch = (x0.cuda(), t.cuda(), y.cuda(), mask.cuda(), noise.cuda())
    step = GraphedTrainStep(m, DDPMEpsLoss(), red, batch)
    l1 = step(*batch).clone()
    g1 = torch.cat([b["flat"].clone() for b in red.buckets])
    assert po.rel_err(l1.cpu().reshape(1), eager.cpu().reshape(1)) < 1e-4
    assert po.rel_err(g1.cpu(), eager_g.cpu()) < 1e-4
    opt.step()
    l2 = step(*batch).clone()
    g2 = torch.cat([b["flat"].clone() for b in red.buckets])
    red.zero_grad()
    eager2 = train_step(m, DDPMEpsLoss(), *batch[:4], noise=batch[4], reducer=red)
    assert not torch.equal(g2, g1)                                # the replay saw the optimizer update
    assert po.rel_err(l2.cpu().reshape(1), eager2.cpu().reshape(1)) < 1e-4
    assert po.rel_err(g2.cpu(), torch.cat([b["flat"] for b in red.buckets]).cpu()) < 1e-4


def test_eager_lora_step_does_not_sync_the_host():
    cfg, sd, m = _setup()
    x0, t, y, mask, noise = (v.cuda() for v in _inputs(cfg))
    red = GradBucketReducer(m)
    opt = FlatAdamW(red, lr=1e-5, weight_decay=1e-2, eps=1e-8)
    loss = DDPMEpsLoss()

    def step():
        red.zero_grad()
        train_step(m, loss, x0, t, y, mask, noise=noise, reducer=red)
        clip_grad_norm_(red, 1.0)
        opt.step()

    step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
