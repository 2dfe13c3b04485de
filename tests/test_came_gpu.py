"""GPU tests (-m gpu) of the fused CAME step (`optim.FlatCAME`, pxa_came_flat) and gradient clipping (`optim.clip_grad_norm_`,
pxa_grad_clip_flat) against the plain-torch restatement of came_pytorch in oracle/came_oracle.py.

Bound: the kernels compute in fp32 with the sums in another order than torch's reductions, so a parameter, exp_avg or
statistic differs from the fp32 oracle by reordered-sum rounding only: normwise relative error <= 1e-5 per tensor (the
differences seen are ~1e-7).  Each test prints its measured errors (shown with `pytest -s` or `-rP`)."""
import pytest
import torch

from oracle import came_oracle as co
from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu
BOUND = 1e-5

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
    from pixart_sigma_b200.optim import FlatAdamW, FlatCAME, clip_grad_norm_
    from pixart_sigma_b200.parallel import GradBucketReducer


def _log(line):
    print(f"[came] {line}")


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


class Odd(torch.nn.Module):
    """Odd sizes at unaligned bucket offsets, 1-row / 1-column matrices, a 4-D conv weight, 2 x 2 matrices, 1-D biases."""

    def __init__(self):
        super().__init__()
        P = torch.nn.Parameter
        self.b0 = P(torch.randn(3))                  # puts everything after it at a 12-byte offset
        self.w = P(torch.randn(37, 53))
        self.row = P(torch.randn(1, 53))
        self.col = P(torch.randn(41, 1))
        self.conv = P(torch.randn(6, 3, 5, 7))
        self.patch = P(torch.randn(300, 4, 2, 2))
        self.big = P(torch.randn(200, 300))
        self.b1 = P(torch.randn(5000))
        self.unused = P(torch.randn(9, 11))         # always a zero gradient


def _pair(seed=0):
    torch.manual_seed(seed)
    a = Odd().cuda()
    ref = [p.detach().clone() for p in a.parameters()]
    return a, ref


def _grads(model, g):
    out = []
    for n, p in model.named_parameters():
        v = torch.zeros_like(p) if n == "unused" else torch.randn(p.shape, generator=g, device="cpu").cuda() * 0.1
        out.append(v)
    return out


def _compare(opt, model, ref, ref_state, tag):
    names = [n for n, _ in model.named_parameters()]
    sd = opt.to_torch_state_dict(model)
    errs = {}
    for k, (n, p) in enumerate(model.named_parameters()):
        errs[n] = _rel(p.detach(), ref[k])
        for key, v in ref_state[k].items():
            if torch.is_tensor(v) and v.dim() > 0:
                errs[f"{n}.{key}"] = _rel(sd["state"][k][key], v)
        errs[f"{n}.RMS"] = _rel(sd["state"][k]["RMS"].reshape(1), torch.as_tensor(ref_state[k]["RMS"]).reshape(1))
    worst = max(errs, key=errs.get)
    _log(f"{tag}: worst {worst} = {errs[worst]:.2e}")
    assert errs[worst] <= BOUND, (worst, errs[worst], names)


@pytest.mark.parametrize("wd", [0.0, 3e-2])
def test_flat_came_matches_oracle_on_odd_shapes(wd):
    model, ref = _pair()
    red = GradBucketReducer(model, bucket_of=lambda n: "a" if n in ("b0", "w", "row", "col") else "b")
    opt = FlatCAME(red, lr=1e-2, weight_decay=wd)
    assert any(e["offset"] % 4 for e in opt.entries)
    states = [{} for _ in ref]
    g = torch.Generator().manual_seed(1)
    for _ in range(5):
        grads = _grads(model, g)
        red.zero_grad()
        for p, v in zip(model.parameters(), grads):
            p.grad.copy_(v)
        opt.step()
        co.came_step(ref, grads, states, lr=1e-2, weight_decay=wd)
    torch.cuda.synchronize()
    _compare(opt, model, ref, states, f"odd shapes wd={wd}")
    assert all(float(b["flat"][-1]) == 0 for b in red.buckets if b["flat"].numel() > sum(p.numel() for p in b["params"]))


@pytest.mark.parametrize("max_norm,grad_scale", [(0.01, 1.0), (1e4, 1.0), (0.05, 0.5), (1e4, 0.5)])
def test_clip_grad_norm_matches_torch(max_norm, grad_scale):
    model, _ = _pair(2)
    red = GradBucketReducer(model, bucket_of=lambda n: n[:1])
    g = torch.Generator().manual_seed(3)
    grads = _grads(model, g)
    for p, v in zip(model.parameters(), grads):
        p.grad.copy_(v)
    params = [torch.nn.Parameter(v.clone()) for v in grads]
    for q, v in zip(params, grads):
        q.grad = v * grad_scale
    want = torch.nn.utils.clip_grad_norm_(params, max_norm)
    got = clip_grad_norm_(red, max_norm, grad_scale=grad_scale)
    assert got.dim() == 0 and got.is_cuda
    assert abs(got.item() - want.item()) <= 1e-5 * want.item(), (got.item(), want.item())
    err = max(_rel(p.grad, q.grad) for p, q in zip(model.parameters(), params) if q.grad.norm() > 0)
    _log(f"clip max_norm={max_norm} grad_scale={grad_scale}: norm {got.item():.6e} vs {want.item():.6e}, grads {err:.2e}")
    assert err <= BOUND


def _state_tensors(opt, model):
    return [p.detach().clone() for p in model.parameters()] + [t.clone() for t in opt.exp_avg] + \
        [getattr(opt, k).clone() for k in opt._STATE]


def test_step_is_deterministic_and_graph_capture_is_bitwise_equal():
    model, _ = _pair(4)
    red = GradBucketReducer(model)
    opt = FlatCAME(red, lr=1e-2, weight_decay=1e-2)
    g = torch.Generator().manual_seed(5)
    for p, v in zip(model.parameters(), _grads(model, g)):
        p.grad.copy_(v)
    grads0 = [b["flat"].clone() for b in red.buckets]
    clip_grad_norm_(red, 0.5)                                             # warm-up: allocates the clip workspace
    opt.step()
    start = opt.state_dict(), [p.detach().clone() for p in model.parameters()]

    def restore():
        opt.load_state_dict(start[0])
        with torch.no_grad():
            for p, v in zip(model.parameters(), start[1]):
                p.copy_(v)
            for b, v in zip(red.buckets, grads0):
                b["flat"].copy_(v)

    def eager():
        restore()
        clip_grad_norm_(red, 0.5)
        opt.step()
        torch.cuda.synchronize()
        return _state_tensors(opt, model)

    r1, r2 = eager(), eager()
    assert all(torch.equal(a, b) for a, b in zip(r1, r2))

    restore()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph):
            norm = clip_grad_norm_(red, 0.5)
            opt.step()
    torch.cuda.current_stream().wait_stream(side)
    restore()
    opt.step_count = start[0]["step"] + 1
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(_state_tensors(opt, model), r1))
    assert torch.isfinite(norm)

    # an lr change between replays takes effect: replay with lr 0 leaves the parameters as they were
    restore()
    opt.lr = 0.0
    before = [p.detach().clone() for p in model.parameters()]
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(p, q) for p, q in zip(model.parameters(), before))
    restore()
    opt.lr = 1e-2
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(_state_tensors(opt, model), r1))


def test_clip_and_step_do_not_sync_the_host():
    model, _ = _pair(6)
    red = GradBucketReducer(model)
    opt = FlatCAME(red)
    for p in model.parameters():
        p.grad.normal_()
    clip_grad_norm_(red, 0.01)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            clip_grad_norm_(red, 0.01)
            opt.step()
        opt.lr = 3e-5
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_xl_parameter_set_matches_oracle():
    """Every parameter of PixArtMS-XL/2 (610.9 M, 29 buckets), two steps against the oracle (~15 GB of device memory)."""
    from pixart_sigma_b200 import PixArtMS_XL_2
    with torch.device("cuda"):
        model = PixArtMS_XL_2(input_size=128)
    red = GradBucketReducer(model)
    opt = FlatCAME(red, lr=1e-3, weight_decay=1e-2)
    ref = [p.detach().clone() for p in model.parameters()]
    states = [{} for _ in ref]
    n0 = lib.launch_count()
    for s in range(2):
        torch.manual_seed(10 + s)
        for p in model.parameters():
            p.grad.normal_().mul_(1e-3)
        clip_grad_norm_(red, 0.01)
        grads = [p.grad.clone() for p in model.parameters()]
        opt.step()
        co.came_step(ref, grads, states, lr=1e-3, weight_decay=1e-2)
        del grads
    torch.cuda.synchronize()
    assert lib.launch_count() - n0 == 2 * (2 + 7)
    worst, wname = 0.0, ""
    sd = opt.to_torch_state_dict(model)
    for k, (n, p) in enumerate(model.named_parameters()):
        for name, a, b in [(n, p.detach(), ref[k])] + [(f"{n}.{key}", sd["state"][k][key], v) for key, v in states[k].items()
                                                       if torch.is_tensor(v) and v.dim() > 0]:
            e = _rel(a, b)
            if e > worst:
                worst, wname = e, name
    _log(f"XL/2 two steps: worst {wname} = {worst:.2e}")
    assert worst <= BOUND, (wname, worst)


def test_training_step_with_clip_and_came_matches_the_oracle_path():
    """depth-2 model: train_step + clip(0.01) + FlatCAME for 3 steps vs the same model with plain autograd gradients, torch's
    clip_grad_norm_ and the oracle's CAME loop, at the Sigma configs' lr.  Both sides run the same forward / backward kernels,
    so the losses differ only by the optimizer's rounding and its effect on later gradients (bound 1e-4 rel.), and so do the
    parameter updates p_3 - p_0 (bound 5e-2 rel., normwise over all parameters: the gradients of the two sides already differ
    by accumulation-order rounding, and a 1-D parameter's first CAME update is sign(g) times a constant)."""
    from oracle.gen_golden_train import train_inputs
    from pixart_sigma_b200 import build_model
    from pixart_sigma_b200.training import IDDPMLoss, train_step
    cfg = po.OracleConfig(depth=2, input_size=32, pe_interpolation=0.5)
    sd = {k: v.to(torch.bfloat16).float() for k, v in po.synthetic_state_dict(cfg, seed=0).items()}
    x0, t, y, mask, noise = train_inputs(cfg, 2, (32, 32), [10, 600], [300, 50])
    args = (x0.cuda(), t.cuda(), y.to(torch.bfloat16).cuda(), mask.cuda())

    def build():
        kw = dict(type="PixArtMS", depth=2, input_size=32, pe_interpolation=0.5, model_max_length=300)
        with torch.device("cuda"):
            m = build_model(kw)
        m.load_state_dict(sd, strict=False)
        m = m.float().train()
        m.y_embedder.uncond_prob = 0.0
        return m

    fused, plain = build(), build()
    red = GradBucketReducer(fused)
    opt = FlatCAME(red, lr=2e-5)
    p0 = [p.detach().clone() for p in plain.parameters()]
    params = [p for p in plain.parameters() if p.requires_grad]
    states = [{} for _ in params]
    loss_f, loss_p = [], []
    for _ in range(3):
        red.zero_grad()
        loss_f.append(train_step(fused, IDDPMLoss(), *args, noise=noise.cuda(), reducer=red).item())
        clip_grad_norm_(red, 0.01)
        opt.step()
        plain.zero_grad(set_to_none=True)
        loss_p.append(train_step(plain, IDDPMLoss(), *args, noise=noise.cuda()).item())
        torch.nn.utils.clip_grad_norm_(params, 0.01)
        co.came_step([p.data for p in params], [p.grad for p in params], states, lr=2e-5)
    lerr = max(abs(a - b) / abs(b) for a, b in zip(loss_f, loss_p))
    da = torch.cat([(a.detach() - q).flatten() for a, q in zip(fused.parameters(), p0)])
    db = torch.cat([(b.detach() - q).flatten() for b, q in zip(plain.parameters(), p0)])
    perr = _rel(da, db)
    _log(f"train_step + clip + CAME, 3 steps: loss rel err {lerr:.2e} ({loss_f} vs {loss_p}), parameter updates {perr:.2e}")
    assert lerr <= 1e-4 and perr <= 5e-2, f"loss rel err {lerr:.3e}, parameter-update rel err {perr:.3e}"


def test_argument_rejection():
    model, _ = _pair(7)
    red = GradBucketReducer(model)
    opt = FlatCAME(red)
    args = opt._args
    args.step = 1
    for field, value, code in [("step", 0, "step"), ("rms", 0, "null"), ("exp_avg_sq", args.exp_avg_sq + 4, "aligned"),
                               ("workspace_bytes", 4, "workspace")]:
        old = getattr(args, field)
        setattr(args, field, value)
        try:
            with pytest.raises(lib.PxaError, match=code):
                lib.came_flat(args)
        finally:
            setattr(args, field, old)
    partials = torch.empty(lib.GRAD_CLIP_PARTS, device="cuda")
    norm = torch.empty((), device="cuda")
    with pytest.raises(lib.PxaError, match="aligned"):
        lib.grad_clip_flat([red.buckets[0]["flat"][1:]], partials, norm, max_norm=1.0)
    with pytest.raises(lib.PxaError):
        lib.grad_clip_flat([red.buckets[0]["flat"].cpu()], partials, norm, max_norm=1.0)
    bf = Odd().cuda().to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="fp32"):
        FlatCAME(GradBucketReducer(bf))
    with pytest.raises(RuntimeError, match="fp32"):
        FlatCAME(GradBucketReducer(Odd()))
    # FlatAdamW and FlatCAME share the clipping entry point
    m2, _ = _pair(8)
    red2 = GradBucketReducer(m2)
    adam = FlatAdamW(red2)
    for p in m2.parameters():
        p.grad.normal_()
    clip_grad_norm_(red2, 1.0)
    adam.step()
    torch.cuda.synchronize()
