"""DoRA on the kernels (-m gpu): pxa_dora_norm, pxa_dora_bwd and the column-scaled GEMM against float64; the DoRA training
forward / backward against the DoRA oracle (tests/dora_oracle.py) in fp32 on the same bf16-rounded weights, as
test_lora_train_gpu.py does for LoRA; optimizer steps, the adapter round trip, graph capture, the absence of host syncs, and
merged sampling.  Model-level bounds are normwise per tensor: loss 2e-3, gradients 2e-2.  The measured values are printed
(pytest -s shows them)."""
import pytest
import torch

import dora_oracle as do
from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import build_model, lib, lora
    from pixart_sigma_b200.graph import GraphedForward
    from pixart_sigma_b200.optim import FlatAdamW, clip_grad_norm_
    from pixart_sigma_b200.parallel import GradBucketReducer
    from pixart_sigma_b200.training import DDPMEpsLoss, GraphedTrainStep, train_step

U = 2.0 ** -24            # fp32 unit roundoff
KINDS = {"plain": ({}, {}),
         "kv_compress": (dict(kv_sampling="conv", kv_scale_factor=2, kv_compress_layer=[0]),
                         dict(kv_compress_config=dict(sampling="conv", scale_factor=2, kv_compress_layer=[0]))),
         "qk_norm": (dict(qk_norm=True), dict(qk_norm=True))}
R = 4


def _log(line):
    print(line)


def _r(v):
    return v.to(torch.bfloat16).float()


# ------------------------------------------------------------------------------------------------- kernels
def _operands(N, K, G, r, s, seed):
    """bf16 W [N, K] and the prepared adapter operands a [T, K], b = s blockdiag(B) [N, T], as lora.prepare_operands builds."""
    g = torch.Generator().manual_seed(seed)
    T = (G * r + 7) // 8 * 8
    W = (torch.randn(N, K, generator=g) * 0.02).to(torch.bfloat16)
    a = torch.zeros(T, K)
    a[:G * r] = torch.randn(G * r, K, generator=g) / r
    b = torch.zeros(N, T)
    Ng = N // G
    for i in range(G):
        b[i * Ng:(i + 1) * Ng, i * r:(i + 1) * r] = s * torch.randn(Ng, r, generator=g) * 0.05
    return W, a.to(torch.bfloat16), b.to(torch.bfloat16), T


@pytest.mark.parametrize("N,K,G", [(1152, 1152, 1), (3456, 1152, 3), (4608, 1152, 1), (1152, 4608, 1)])
@pytest.mark.parametrize("r", [16, 5])
def test_dora_norm_against_fp64(N, K, G, r):
    """wn = ||W + b a||_row against float64 of the same bf16 operands.  Each element e = w + sum_t b a is formed with T fp32
    fmas: |de| <= (T + 1) u (|w| + sum_t |b a|); the squares run as one fmaf chain per lane over K / 64 slices (two
    elements per step) and a 5-level shuffle tree, then sqrtf: |d wn| <= ||de||_row + (K / 64 + 8) u wn.  c = m / wn adds
    one rounding."""
    W, a, b, T = _operands(N, K, G, r, 2.0, seed=N + K + r)
    m = torch.rand(N) + 0.5
    wn, c = torch.empty(N, device="cuda"), torch.empty(N, device="cuda")
    lib.dora_norm([(W.cuda(), a.cuda(), b.cuda(), m.cuda(), wn, c)], N=N, K=K, T=T)
    wd, ad, bd = W.double(), a.double(), b.double()
    e = wd + bd @ ad
    ref = e.norm(dim=1)
    de = (T + 1) * U * (wd.abs() + bd.abs() @ ad.abs())
    bound = de.norm(dim=1) + (K / 64 + 8) * U * ref
    err = (wn.double().cpu() - ref).abs()
    cref = m.double() / ref
    cerr = (c.double().cpu() - cref).abs()
    cbound = cref * (bound / ref + 2 * U)
    _log(f"dora_norm N={N} K={K} G={G} r={r}: max err / bound wn {(err / bound).max():.3f}, c {(cerr / cbound).max():.3f}")
    assert (err <= bound).all() and (cerr <= cbound).all()
    # deterministic, and B = 0 with m = wn gives c = 1 exactly
    wn2 = torch.empty(N, device="cuda")
    lib.dora_norm([(W.cuda(), a.cuda(), b.cuda(), None, wn2, None)], N=N, K=K, T=T)
    assert torch.equal(wn, wn2)
    z = torch.zeros_like(b).cuda()
    w0 = torch.empty(N, device="cuda")
    lib.dora_norm([(W.cuda(), a.cuda(), z, None, w0, None)], N=N, K=K, T=T)
    c1 = torch.empty(N, device="cuda")
    lib.dora_norm([(W.cuda(), a.cuda(), z, w0, None, c1)], N=N, K=K, T=T)
    assert torch.equal(c1, torch.ones_like(c1))


def test_dora_norm_batches_more_items_than_one_launch_holds():
    """84 same-shaped items (the 1152 x 1152 group of XL/2) run over two launches; each item's result is its own."""
    N = K = 1152
    items, refs = [], []
    for i in range(84):
        W, a, b, T = _operands(N, K, 1, 4, 2.0, seed=i)
        wn = torch.empty(N, device="cuda")
        items.append((W.cuda(), a.cuda(), b.cuda(), None, wn, None))
        refs.append((W.double() + b.double() @ a.double()).norm(dim=1))
    lib.dora_norm(items, N=N, K=K, T=8)
    err = max(float(((it[4].double().cpu() - ref) / ref).abs().max()) for it, ref in zip(items, refs))
    assert err < 1e-5, err


@pytest.mark.parametrize("M,N", [(4096, 1152), (1000, 3456), (77, 2304)])
def test_dora_bwd_against_fp64_deterministic_and_aliased(M, N):
    """dz = bf16(c g): one fp32 product then the bf16 rounding, <= 2^-8 |c g| + u |c g|.  dm = sum_r g (y - b) / m: each term
    one subtraction and one fma, 16-row chains per thread, an 8-term smem sum per chunk and the ordered sum over the chunks,
    then the division: |d dm| <= (16 + 8 + chunks + 4) u sum_r |g (y - b)| / |m|."""
    g0 = torch.Generator().manual_seed(M + N)
    g = torch.randn(M, N, generator=g0).to(torch.bfloat16)
    y = torch.randn(M, N, generator=g0).to(torch.bfloat16)
    bias = (torch.randn(N, generator=g0) * 0.1).to(torch.bfloat16)
    c = torch.rand(N, generator=g0) + 0.5
    m = torch.rand(N, generator=g0) + 0.5
    dm0 = torch.randn(N, generator=g0)
    dz = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    dm = dm0.clone().cuda()
    lib.dora_bwd(g.cuda(), y.cuda(), bias.cuda(), c.cuda(), m.cuda(), dz, dm)
    gd, yd, bd = g.double(), y.double(), bias.double()
    ref_dz = c.double() * gd
    assert ((dz.double().cpu() - ref_dz).abs() <= (2.0 ** -8 + U) * ref_dz.abs()).all()
    prod = gd * (yd - bd)
    ref_dm = dm0.double() + prod.sum(0) / m.double()
    chunks = (M + lib.DORA_BWD_ROWS - 1) // lib.DORA_BWD_ROWS
    bound = (16 + 8 + chunks + 4) * U * prod.abs().sum(0) / m.double() + U * ref_dm.abs()
    err = (dm.double().cpu() - ref_dm).abs()
    _log(f"dora_bwd M={M} N={N}: max err / bound dm {(err / bound).max():.3f}")
    assert (err <= bound).all()
    # two launches give the same bits; dz over g gives the same dz and dm
    dm2 = dm0.clone().cuda()
    dz2 = torch.empty_like(dz)
    lib.dora_bwd(g.cuda(), y.cuda(), bias.cuda(), c.cuda(), m.cuda(), dz2, dm2)
    assert torch.equal(dz, dz2) and torch.equal(dm, dm2)
    ga = g.cuda()
    dm3 = dm0.clone().cuda()
    lib.dora_bwd(ga, y.cuda(), bias.cuda(), c.cuda(), m.cuda(), ga, dm3)
    assert torch.equal(ga, dz) and torch.equal(dm3, dm)


FORMS = ["bias", "gelu", "gelu_aux", "res_bf16", "res_f32_gate_branch"]


def _gemm_case(form, M, N, K, T, seed):
    g = torch.Generator().manual_seed(seed)
    d = lambda *s, std=1.0: (torch.randn(*s, generator=g) * std).to(torch.bfloat16).cuda()
    x, w, bias = d(M, K), d(N, K, std=0.03), d(N, std=0.1)
    tail = (d(M, T), d(N, T, std=0.03)) if T else None
    kw, out_dt = {}, torch.bfloat16
    if form == "gelu":
        kw["epilogue"] = lib.EPI_BIAS_GELU
    elif form == "gelu_aux":
        kw.update(epilogue=lib.EPI_BIAS_GELU_AUX)
    elif form == "res_bf16":
        kw.update(epilogue=lib.EPI_BIAS_RESIDUAL, residual=d(M, N))
    elif form == "res_f32_gate_branch":
        out_dt = torch.float32
        kw.update(epilogue=lib.EPI_BIAS_RESIDUAL, residual=torch.randn(M, N, generator=g).cuda(),
                  gate=(torch.randn(2, N, generator=g) * 0.5).cuda(), gate_batch_stride=N, rows_per_batch=M // 2,
                  aux_is_branch=True)
    return x, w, bias, tail, kw, out_dt


def _run(x, w, bias, tail, kw, out_dt, M, N, col_scale=None, w_scale=None):
    out = torch.empty(M, N, dtype=out_dt, device="cuda")
    aux = torch.empty(M, N, dtype=torch.bfloat16, device="cuda") if kw.get("epilogue") in (lib.EPI_BIAS_GELU_AUX,) or \
        kw.get("aux_is_branch") else None
    if w_scale is not None:                               # scale the weight rows instead (exact for powers of two)
        w = (w.float() * w_scale[:, None]).to(torch.bfloat16)
        tail = None if tail is None else (tail[0], (tail[1].float() * w_scale[:, None]).to(torch.bfloat16))
    tkw = {} if tail is None else dict(tail_a=tail[0], tail_w=tail[1])
    lib.gemm(x, w, bias, out, out_aux=aux, col_scale=col_scale, **kw, **tkw)
    return out, aux


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("T", [0, 16])
def test_gemm_dora_scale_is_exact_on_powers_of_two(form, T):
    """With c a power of two per column, c acc is exact in fp32 and equals the accumulator of the row-scaled weights (each
    product scales exactly): the column-scaled GEMM must then be bit for bit the unscaled GEMM on c W (and c tail_w) -- the
    kernel whose every epilogue test_gemm_numerics_gpu.py bounds against float64."""
    M, N, K = 512, 1152, 1152
    x, w, bias, tail, kw, out_dt = _gemm_case(form, M, N, K, T, seed=7)
    kw["block_n"] = 128                                  # the same tiling for every run compared
    c = 2.0 ** torch.randint(-3, 4, (N,), generator=torch.Generator().manual_seed(1)).float().cuda()
    got, got_aux = _run(x, w, bias, tail, kw, out_dt, M, N, col_scale=c)
    want, want_aux = _run(x, w, bias, tail, kw, out_dt, M, N, w_scale=c)
    assert torch.equal(got, want)
    assert got_aux is None or torch.equal(got_aux, want_aux)
    one, _ = _run(x, w, bias, tail, kw, out_dt, M, N, col_scale=torch.ones(N, device="cuda"))
    base, _ = _run(x, w, bias, tail, kw, out_dt, M, N)
    assert torch.equal(one, base)                         # c = 1 is the unscaled GEMM


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("T", [0, 16])
def test_gemm_dora_against_fp64(form, T):
    """A general c against float64: y = c (x W^T + tail) + bias in float64 through the epilogue.  Bound per element: the
    accumulator's K 2^-23 sum |a w| allowance times |c|, u |y| for the scaling and bias add, then the output's rounding (one
    bf16 ulp, two for GELU, whose own contract is one ulp) -- looser than gemm_bounds.py's, which the power-of-two test
    inherits exactly."""
    M, N, K = 384, 1152, 1152
    x, w, bias, tail, kw, out_dt = _gemm_case(form, M, N, K, T, seed=11)
    c = (torch.rand(N, generator=torch.Generator().manual_seed(2)) + 0.5).cuda()
    got, aux = _run(x, w, bias, tail, kw, out_dt, M, N, col_scale=c)
    xd, wd = x.double(), w.double()
    acc = xd @ wd.T
    absacc = xd.abs() @ wd.abs().T
    if tail is not None:
        acc = acc + tail[0].double() @ tail[1].double().T
        absacc = absacc + tail[0].double().abs() @ tail[1].double().abs().T
    cd = c.double()
    y = cd * acc + bias.double()
    slack = cd * (K + T) * 2.0 ** -23 * absacc + U * y.abs()
    ulp = lambda v, dt: v.abs().clamp_min(1e-30) * (2.0 ** -7 if dt == torch.bfloat16 else 2.0 ** -23)
    gelu = lambda v: 0.5 * v * (1 + torch.tanh(0.7978845608028654 * (v + 0.044715 * v ** 3)))
    if form == "bias":
        ref, tol = y, slack + ulp(y, torch.bfloat16)
    elif form in ("gelu", "gelu_aux"):
        ref = gelu(y)
        tol = 1.2 * slack + 2 * ulp(ref, torch.bfloat16) + 1e-30
        if form == "gelu_aux":
            assert ((aux.double() - y).abs() <= slack + ulp(y, torch.bfloat16)).all()
    elif form == "res_bf16":
        ref = kw["residual"].double() + y
        tol = slack + ulp(ref, torch.bfloat16) + U * ref.abs()
    else:
        gt = kw["gate"].double().repeat_interleave(M // 2, 0)
        ref = kw["residual"].double() + gt * y
        tol = gt.abs() * slack + ulp(ref, torch.float32)
        assert ((aux.double() - y).abs() <= slack + ulp(y, torch.bfloat16)).all()   # the branch output c acc + b
    err = (got.double() - ref).abs()
    _log(f"gemm dora {form} T={T}: max err / bound {(err / tol).max():.3f}")
    assert (err <= tol).all()


def test_gemm_dora_rejects_other_forms():
    x = torch.zeros(128, 64, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(128, 64, dtype=torch.bfloat16, device="cuda")
    c = torch.ones(128, device="cuda")
    with pytest.raises(lib.PxaError, match="column scale"):
        lib.gemm(x, w, None, torch.empty(128, 128, dtype=torch.bfloat16, device="cuda"), epilogue=lib.EPI_MUL_DGELU,
                 residual=torch.zeros(128, 128, dtype=torch.bfloat16, device="cuda"), col_scale=c)


# ------------------------------------------------------------------------------------------------- the model
def _setup(kind="plain", ckpt=False, fresh=False, seed=0):
    """A depth-2 fp32 model on bf16-rounded weights with a rank-4 DoRA adapter: bf16-representable A and (unless fresh) B,
    and a magnitude 10 % off ||W|| (so that c != 1)."""
    ckw, mkw = KINDS[kind]
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5, **ckw)
    sd = {k: _r(v) for k, v in po.synthetic_state_dict(cfg, seed=3).items()}
    kw = dict(type="PixArtMS", depth=2, input_size=32, pe_interpolation=0.5, model_max_length=300, class_dropout_prob=0.0, **mkw)
    with torch.device("cuda"):
        m = build_model(kw, use_grad_checkpoint=ckpt)
    m.load_state_dict(sd, strict=False)
    m = m.float().train()
    lora.inject_dora(m, R, generator=torch.Generator().manual_seed(seed))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for _, mod in lora._adapted(m):
            mod.lora_A.copy_(_r(mod.lora_A))
            if not fresh:
                mod.lora_B.copy_(_r(torch.randn(mod.lora_B.shape, generator=g) * 0.02))
                mod.lora_magnitude.mul_((1 + 0.1 * torch.randn(mod.lora_magnitude.shape, generator=g)).cuda())
    return cfg, sd, m


def _inputs(cfg):
    x, _, y, mask = po.synthetic_inputs(cfg, 2, (32, 32), lens=[300, 77])
    g = torch.Generator().manual_seed(5)
    return x * 0.5, torch.tensor([17, 803]), _r(y), mask, torch.randn(x.shape, generator=g)


def _native_loss(m, loss, x0, t, y, mask, noise):
    kw = dict(y=y.cuda(), mask=mask.cuda(), data_info=None)
    return loss.training_losses(m, x0.cuda(), t.cuda(), kw, noise=noise.cuda())["loss"].mean()


def _oracle_adapters(m):
    return {n: tuple(getattr(mod, k).detach().float().cpu().clone().requires_grad_() for k in ("lora_A", "lora_B", "lora_magnitude"))
            for n, mod in lora._adapted(m)}


def _oracle_loss(sd, ad, cfg, x0, t, y, mask, noise):
    fn = lambda xx, timestep, **kw: do.forward_grad(sd, ad, 2.0, cfg, xx, timestep.float(), kw["y"], mask=kw["mask"])
    return DDPMEpsLoss().training_losses(fn, x0, t, dict(y=y, mask=mask), noise=noise)["loss"].mean()


TRAINABLE = (".lora_A", ".lora_B", ".lora_magnitude")


def test_fresh_adapter_is_bitwise_the_base_forward_and_trains_only_the_adapter():
    cfg, sd, m = _setup(fresh=True)
    x0, t, y, mask, noise = _inputs(cfg)
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
    bucketed = {names[id(p)] for b in red.buckets for p in b["params"]}
    assert all(n.endswith(TRAINABLE) for n in bucketed)
    assert bucketed == {n for n, p in m.named_parameters() if p.requires_grad}
    assert any(n.endswith(".lora_magnitude") for n in bucketed)
    assert all(p.grad is None for n, p in m.named_parameters() if not n.endswith(TRAINABLE))
    assert any(p.grad.abs().sum() > 0 for n, p in m.named_parameters() if n.endswith(".lora_magnitude"))


@pytest.mark.parametrize("kind", list(KINDS))
def test_adapter_gradients_match_oracle(kind):
    """Every adapter's A, B and magnitude gradient against the oracle's autograd; checkpointing on and off agree to 1e-4."""
    grads = {}
    for ckpt in (False, True):
        cfg, sd, m = _setup(kind, ckpt=ckpt)
        x0, t, y, mask, noise = _inputs(cfg)
        loss = _native_loss(m, DDPMEpsLoss(), x0, t, y, mask, noise)
        loss.backward()
        grads[ckpt] = {n + "." + k: getattr(mod, k).grad.float().cpu() for n, mod in lora._adapted(m)
                       for k in ("lora_A", "lora_B", "lora_magnitude")}
    ad = _oracle_adapters(m)
    want = _oracle_loss(sd, ad, cfg, x0, t, y, mask, noise)
    want.backward()
    lerr = po.rel_err(loss.detach().cpu().reshape(1), want.detach().reshape(1))
    errs = {}
    for n, (A, B, mg) in ad.items():
        for k, p in (("lora_A", A), ("lora_B", B), ("lora_magnitude", mg)):
            errs[n + "." + k] = po.rel_err(grads[False][n + "." + k], p.grad)
    ck = max(po.rel_err(grads[True][k], grads[False][k]) for k in grads[False])
    worst = max(errs, key=errs.get)
    wm = max((k for k in errs if k.endswith("magnitude")), key=errs.get)
    _log(f"dora grads {kind}: loss {lerr:.2e}, max grad {errs[worst]:.2e} ({worst}), max magnitude grad {errs[wm]:.2e} ({wm}), "
         f"ckpt on/off {ck:.2e}")
    for must in ("x_embedder.proj", "y_embedder.y_proj.fc1", "t_block.1", "final_layer.linear", "blocks.0.attn.qkv",
                 "blocks.1.cross_attn.kv_linear", "blocks.0.cross_attn.proj", "blocks.1.mlp.fc2"):
        assert must + ".lora_magnitude" in errs
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
    p0 = {n: tuple(v.detach().clone() for v in vs) for n, vs in ad.items()}
    red = GradBucketReducer(m)
    opt = FlatAdamW(red, lr=1e-5, weight_decay=1e-2, eps=1e-8)
    _steps(m, red, opt, x0, t, y, mask, noise)
    params = [p for vs in ad.values() for p in vs]
    topt = torch.optim.AdamW(params, lr=1e-5, weight_decay=1e-2, eps=1e-8)
    for _ in range(3):
        topt.zero_grad()
        _oracle_loss(sd, ad, cfg, x0, t, y, mask, noise).backward()
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        topt.step()
    keys = ("lora_A", "lora_B", "lora_magnitude")
    got = torch.cat([(getattr(mod, k).detach().cpu() - p0[n][i]).flatten() for n, mod in lora._adapted(m) for i, k in enumerate(keys)])
    want = torch.cat([(ad[n][i].detach() - p0[n][i]).flatten() for n, _ in lora._adapted(m) for i in range(3)])
    err = po.rel_err(got, want)
    _log(f"dora 3 AdamW steps: update rel_err {err:.2e}")
    # the LoRA test's bound (test_lora_train_gpu.py): Adam's per-element normalisation amplifies the gradients' bf16 error
    # on elements whose gradient is near zero
    assert err < 1e-1, err


def test_adapter_round_trip_after_training(tmp_path):
    """save_adapter -> fresh model -> load_dora_adapter -> merge_lora: its no-grad forward matches the trained model's
    unmerged training forward (1e-2); the trained adapter moves the output by more than 10x that."""
    cfg, sd, m = _setup(fresh=True)
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
    lora.load_dora_adapter(f, str(tmp_path))
    lora.merge_lora(f)
    f = f.to(torch.bfloat16).eval()
    with torch.no_grad():
        merged = f(x0.cuda(), t.cuda(), **kw).float().cpu()
    err, moved = po.rel_err(merged, trained), po.rel_err(base, trained)
    _log(f"dora round trip: merged vs trained {err:.2e}, adapter moves the output by {moved:.2e}")
    assert err < 1e-2 and moved > 10 * err, (err, moved)


def test_graphed_dora_step_matches_eager_and_sees_updates():
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
    # only the magnitudes move: a replay must see them (c is recomputed inside the graph)
    with torch.no_grad():
        for _, mod in lora._adapted(m):
            mod.lora_magnitude.mul_(1.05)
    l2 = step(*batch).clone()
    g2 = torch.cat([b["flat"].clone() for b in red.buckets])
    red.zero_grad()
    eager2 = train_step(m, DDPMEpsLoss(), *batch[:4], noise=batch[4], reducer=red)
    assert not torch.equal(g2, g1) and not torch.equal(l2, l1)
    assert po.rel_err(l2.cpu().reshape(1), eager2.cpu().reshape(1)) < 1e-4
    assert po.rel_err(g2.cpu(), torch.cat([b["flat"] for b in red.buckets]).cpu()) < 1e-4
    opt.step()
    l3 = step(*batch).clone()
    red.zero_grad()
    eager3 = train_step(m, DDPMEpsLoss(), *batch[:4], noise=batch[4], reducer=red)
    assert po.rel_err(l3.cpu().reshape(1), eager3.cpu().reshape(1)) < 1e-4


def test_eager_dora_step_does_not_sync_the_host():
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


def test_merged_sampling_matches_oracle_unmerged_and_unmerge_restores():
    """Unmerge restores the weights bit for bit; a merged DoRA model on bf16 weights, its no-grad forward and its GraphedForward
    replay, against the oracle's UNMERGED DoRA forward (1e-2, the merged-LoRA bound of test_lora_gpu.py)."""
    cfg, sd, m = _setup()
    x0, t, y, mask, _ = _inputs(cfg)
    ad = {n: tuple(v.detach() for v in vs) for n, vs in _oracle_adapters(m).items()}
    want = do.forward(sd, ad, 2.0, cfg, x0, t.float(), y, mask=mask)
    before = {k: v.clone() for k, v in m.state_dict().items()}
    m = m.eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="merge_lora"):
        m(x0.cuda(), t.cuda(), y.cuda(), mask=mask.cuda())
    lora.merge_lora(m)                                    # in fp32, then sampled on bf16 weights
    lora.unmerge_lora(m)
    after = m.state_dict()
    assert all(torch.equal(after[k], v) for k, v in before.items())
    lora.merge_lora(m)
    m = m.to(torch.bfloat16)
    with torch.no_grad():
        got = m(x0.cuda(), t.cuda(), y.cuda(), mask=mask.cuda()).float().cpu()
    gf = GraphedForward(m, "forward")
    graphed = gf(x0.cuda(), t.cuda(), y.cuda(), mask.cuda()).float().cpu()
    base = po.forward(sd, cfg, x0, t.float(), y, mask=mask)
    err, gerr, moved = po.rel_err(got, want), po.rel_err(graphed, want), po.rel_err(base, want)
    _log(f"dora merged sampling: eager {err:.2e}, graphed {gerr:.2e} vs the unmerged oracle; the adapter moves it by {moved:.2e}")
    assert err < 1e-2 and gerr < 1e-2 and moved > 10 * err
