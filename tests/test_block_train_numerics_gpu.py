"""The training block (`autograd.BlockFn`) kernel by kernel against float64 (-m gpu), with the stage references of
block_stages.py (whose CPU test proves they compose to float64 autograd of the oracle block).

Each case runs the real BlockFn forward and backward with `autograd.lib` replaced by a recorder that snapshots the output
arguments of every call before and after it.  Then:
  - the recorded call sequence must equal `block_stages.expected_trace` (transposes of the weight shadows aside);
  - every accumulating output must have held, before its kernel, what the test pre-filled (the bucket views) or zero;
  - under activation checkpointing the recomputed forward must equal the first forward bit for bit;
  - every stage's output must lie within its kernel's own bound of the float64 reference formed from the test's weights,
    mod, dout, captions and the earlier stages' outputs in their correct roles (with -s: per stage the largest error /
    bound, the fraction correctly rounded and the bias);
  - the gradients BlockFn hands back (x, mod, the caption rows, every parameter's .grad) must be, bit for bit, the stage
    outputs that should land there.
The end-to-end errors against float64 autograd of the oracle block (on the bf16 weights the kernels read) are printed,
not asserted, with the residual path taken out of x.grad (x.grad - dout): the record next to test_training_gpu's 2e-2.

Cases: (1) the benchmarked c5 block: B = 4, a 64 x 64 grid, the model's unpacked caption layout (kv_off None, 300 rows
per sample, kv_len 300, 120, 1, 0), fp32 master weights off the bf16 grid, fp32_attention, activation checkpointing, and
gradients accumulated into pre-filled GradBucketReducer bucket views; (2) the same geometry with bf16 parameters, no
fp32_attention, no checkpointing and gradients through autograd; (3) qk_norm with fp32 norm weights off the bf16 grid
(2 x 32 x 32).  Mutation checks plant wrong wiring in one call (add_in dropped, the shift / scale columns swapped, the
fp32 norm weight in the qk-norm backward) and the stage check must fail at that stage.  (4) The packed caption layout
through PixArtMSBlock.forward (B = 3, 24 x 40, lens 300 / 77 / 9) with one sample's gate_msa and another's gate_mlp
exactly 0.  (5) Parameter-free KV compression: 'ave' on 15 x 17 and 'uniform' on 32 x 32.

Not covered here: the 'conv' KV compression (its fused conv + LayerNorm forward has no element-wise contract yet), LoRA
adapters, and the model's caption projector / final layer around the blocks.

The float64 references are computed on the GPU over all rows (no subsampling).
"""
import time

import pytest
import torch

import block_stages as bs
import gemm_bounds as gb
from oracle import pixart_oracle as po

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import autograd as ag
    from pixart_sigma_b200 import build_model, lib
    from pixart_sigma_b200.parallel import GradBucketReducer

C, H = 1152, 16
# the output arguments (position or keyword) of each lib function BlockFn calls
OUTS = {"ln_modulate": (3,), "gemm": (3, "out_aux"), "flash_attn": (3, "lse"), "layernorm_affine_": (0,),
        "gate_residual_bwd": (3, 4), "gate_residual_fwd": (3,), "gemm_wgrad": (2,), "colsum": (1,),
        "ln_modulate_bwd": (3, 4, 5), "flash_attn_bwd": (6, 7, 8), "transpose": ()}


class Recorder:
    """Stands in for the `lib` module: forwards every call, snapshotting its output arguments (OUTS) before and after it.
    `mutate(name, n, args, kwargs)`, n the call's index among those to `name`, may return changed (args, kwargs)."""

    def __init__(self, mutate=None):
        self.trace, self.mutate, self.count = [], mutate, {}

    def __getattr__(self, name):
        attr = getattr(lib, name)
        if not callable(attr) or name.isupper():
            return attr

        def call(*args, **kwargs):
            n = self.count.get(name, 0)
            self.count[name] = n + 1
            args = list(args)
            if self.mutate is not None:
                args, kwargs = self.mutate(name, n, args, kwargs)
            get = lambda k: args[k] if isinstance(k, int) else kwargs.get(k)
            slots = [k for k in OUTS.get(name, ()) if get(k) is not None]
            before = {k: get(k).clone() for k in slots}
            res = attr(*args, **kwargs)
            if name != "transpose":
                self.trace.append((name, before, {k: get(k).clone() for k in slots}))
            return res
        return call


def _block(qk_norm, dtype, seed=7, sampling=None):
    cfg = po.OracleConfig(depth=1, qk_norm=qk_norm)
    kw = dict(type="PixArtMS", depth=1, input_size=32, pe_interpolation=0.5, model_max_length=300, qk_norm=qk_norm)
    if sampling is not None:                                         # parameter-free: no extra weights
        kw["kv_compress_config"] = dict(sampling=sampling, scale_factor=2, kv_compress_layer=[0])
    with torch.device("cuda"):
        m = build_model(kw)
    sd = po.synthetic_state_dict(cfg, seed=seed)                     # fp32, off the bf16 grid
    m.load_state_dict(sd, strict=False)
    return m.to(dtype).train().blocks[0]


def _run(blk, B, hw, L, lens, *, ckpt, fp32_p, bucket, mutate=None, seed=11, packed=False, zero_gates=()):
    """One BlockFn forward + backward under the recorder; returns everything the checks need.  packed=False: straight
    through `block_train` with the model's unpacked caption layout (L rows per sample, kv_off None); packed=True: through
    PixArtMSBlock.forward with packed captions (mask = lens), mod = scale_shift_table + t, and the gates (sample, column)
    of `zero_gates` exactly 0 (what drop path makes of a dropped sample)."""
    N = hw[0] * hw[1]
    M = B * N
    for mod_ in blk.modules():
        mod_.fp32_attention = fp32_p
    g = torch.Generator(device="cuda").manual_seed(seed)
    x32 = torch.randn(M, C, generator=g, device="cuda").requires_grad_(True)
    cond = torch.randn(B * L, C, generator=g, device="cuda").to(torch.bfloat16).requires_grad_(True)
    mod = (0.3 * torch.randn(B, 6, C, generator=g, device="cuda")).requires_grad_(True)
    dout = torch.randn(M, C, generator=g, device="cuda")
    kv_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
    red = None
    blk.zero_grad(set_to_none=True)
    if bucket:
        red = GradBucketReducer(blk)
        for b_ in red.buckets:
            b_["flat"].copy_(torch.randn(b_["flat"].shape, generator=g, device="cuda"))
    pre = {n: (p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p, dtype=torch.float32))
           for n, p in blk.named_parameters()}
    if packed:
        blk.grad_checkpointing = ckpt
        x = x32.detach().view(B, N, C).requires_grad_(True)
        y = torch.randn(1, sum(lens), C, generator=g, device="cuda").requires_grad_(True)
        t = mod.detach().clone()
        for b, j in zero_gates:                                      # table + (-table) is exactly 0 in fp32
            t[b, j] = -blk.scale_shift_table.detach()[j]
        t = t.reshape(B, 6 * C).requires_grad_(True)
        keys = [(sum(lens[:b]), n) for b, n in enumerate(lens)]
    else:
        keys = [(b * L, n) for b, n in enumerate(lens)]
    rec = Recorder(mutate)
    old = ag.lib
    ag.lib = rec
    try:
        if packed:
            out = blk(x, y, t, lens, hw)
        else:
            out = ag.block_train(blk, x32, cond, kv_len, None, L, mod, B, N, hw, ckpt)
        out.backward(dout.view(out.shape))
        torch.cuda.synchronize()
    finally:
        ag.lib = old
    if red is not None:
        red.remove()
    if packed:
        mod = (blk.scale_shift_table.detach().float()[None] + t.detach().view(B, 6, C)).contiguous()
        vals = dict(x=x.detach().view(M, C), cond=y.detach().view(-1, C).to(torch.bfloat16), mod=mod,
                    gx=x.grad.view(M, C), gmod=t.grad.view(B, 6, C), gcond=y.grad.view(-1, C))
    else:
        vals = dict(x=x32.detach(), cond=cond.detach(), mod=mod.detach(), gx=x32.grad, gmod=mod.grad, gcond=cond.grad)
    return dict(blk=blk, B=B, N=N, keys=keys, lens=lens, hw=hw, dout=dout, pre=pre, rec=rec, ckpt=ckpt, fp32_p=fp32_p,
                bucket=bucket, **vals)


def _inputs(r):
    blk, B, N = r["blk"], r["B"], r["N"]
    d = lambda t: t.detach().double()
    w16 = lambda t: t.detach().to(torch.bfloat16).double()          # the bf16 value a kernel reads of a parameter
    mods = {t: blk.get_submodule(bs.MODULE[t]) for t in bs.TAGS}
    a = blk.attn
    qk = None
    if not isinstance(a.q_norm, torch.nn.Identity):
        qk = {j: (w16(getattr(a, j + "_norm").weight), w16(getattr(a, j + "_norm").bias)) for j in "qk"}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert blk.norm1.eps == blk.norm2.eps and (qk is None or a.q_norm.eps == a.k_norm.eps)
    kv_pick = (a.sampling, a.sr_ratio, r["hw"]) if a.sr_ratio > 1 else None
    pre = {}
    for t in bs.TAGS:
        pre["dW." + t] = d(r["pre"][bs.MODULE[t] + ".weight"])
        pre["db." + t] = d(r["pre"][bs.MODULE[t] + ".bias"])
    return dict(x=d(r["x"]), cond=d(r["cond"]), mod=d(r["mod"]), dout=d(r["dout"]), B=B, N=N, H=H, keys=r["keys"],
                W={t: w16(mods[t].weight) for t in bs.TAGS}, bias={t: w16(mods[t].bias) for t in bs.TAGS}, qk=qk,
                qk_eps=a.q_norm.eps if qk is not None else None, ln_eps=blk.norm1.eps, kv_pick=kv_pick, fp32_p=r["fp32_p"],
                pre=pre,
                splits=lambda m, n, k: gb.auto_splits(m, n, k, sms), cast=lambda t: t.to(torch.bfloat16).double())


def _roles(r):
    qk = not isinstance(r["blk"].attn.q_norm, torch.nn.Identity)
    return bs.roles_of(r["rec"].trace, bs.expected_trace(qk, r["ckpt"]))


def _check(r, name):
    """Every check of the module docstring but the end-to-end print.  Returns the stage tallies."""
    t0 = time.time()
    blk, inp = r["blk"], _inputs(r)
    R, before = _roles(r)
    print(f"\n{name}: {len(r['rec'].trace)} kernel calls recorded")
    for role, p in inp["pre"].items():                               # accumulators held the pre-filled value (or 0)
        assert torch.equal(before[role].double(), p), f"{role}: accumulated onto the wrong values"
    for role in [k for k in before if k.startswith("dm") or k.startswith("dw.") or k.startswith("db.")]:
        if role not in inp["pre"]:
            assert (before[role] == 0).all(), f"{role}: not zero-filled"
    if r["ckpt"]:
        for role in [k for k in R if k.startswith("rc.")]:
            assert torch.equal(R[role], R[role[3:]]), f"checkpoint recompute of {role[3:]} differs from the forward"
    st = bs.BlockStages(inp)
    tallies = st.run(R)
    for t in tallies.values():
        t.report()
    # the gradients BlockFn returned are the stage outputs, bit for bit
    assert torch.equal(r["gx"], R["dx"]), "x.grad"
    assert torch.equal(r["gmod"], torch.stack([R[f"dm{j}"] for j in range(6)], 1)), "mod.grad"
    assert torch.equal(r["gcond"], R["dcond"].to(r["gcond"].dtype)), "caption grad"
    named = dict(blk.named_parameters())
    for t in bs.TAGS:
        for kind, role in (("weight", "dW." + t), ("bias", "db." + t)):
            p = named[bs.MODULE[t] + "." + kind]
            assert torch.equal(p.grad, R[role].to(p.dtype)), f"{t}.{kind}.grad"
    if inp["qk"] is not None:
        for j in "qk":
            for kind, role in (("weight", f"dw.{j}_norm"), ("bias", f"db.{j}_norm")):
                p = named[f"attn.{j}_norm.{kind}"]
                g = R[role].view(C)                                  # through autograd: added onto a bucket view
                g = r["pre"][f"attn.{j}_norm.{kind}"] + g if r["bucket"] else g
                assert torch.equal(p.grad, g.to(p.dtype)), f"{j}_norm.{kind}.grad"
    print(f"{name}: checks took {time.time() - t0:.1f} s")
    return tallies


def _end_to_end(r, name):
    """Print the normwise errors of the returned gradients against float64 autograd of the oracle block."""
    inp = _inputs(r)
    B, N, lens = r["B"], r["N"], r["lens"]
    sd = {"b.scale_shift_table": torch.zeros(6, C, dtype=torch.float64, device="cuda")}
    for t in bs.TAGS:
        sd[f"b.{bs.MODULE[t]}.weight"], sd[f"b.{bs.MODULE[t]}.bias"] = inp["W"][t], inp["bias"][t]
    if inp["qk"] is not None:
        for j in "qk":
            sd[f"b.attn.{j}_norm.weight"], sd[f"b.attn.{j}_norm.bias"] = inp["qk"][j]
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    x = inp["x"].view(B, N, C).clone().requires_grad_(True)
    valid = torch.cat([torch.arange(k0, k0 + n, device="cuda") for k0, n in r["keys"]])
    y = inp["cond"][valid].clone().requires_grad_(True)
    t0 = inp["mod"].reshape(B, 6 * C).clone().requires_grad_(True)
    kvp = inp["kv_pick"]
    out = po.block_forward(sd, "b", x, y[None], t0, lens, r["hw"], H, kvp[1] if kvp else 1, kvp[0] if kvp else None,
                           inp["qk"] is not None)
    out.backward(inp["dout"].view(B, N, C))
    rel = lambda a, b: ((a.double() - b).norm() / b.norm()).item()
    errs = {"x - dout": rel(r["gx"] - r["dout"].view(B * N, C), (x.grad.reshape(B * N, C) - inp["dout"])),
            "mod": rel(r["gmod"], t0.grad.view(B, 6, C)), "caption": rel(r["gcond"][valid], y.grad)}
    named = dict(r["blk"].named_parameters())
    for k, v in sd.items():
        # the k_norm bias moves all logits of a query alike: its exact gradient is 0, so no relative error is printed
        if k not in ("b.scale_shift_table", "b.attn.k_norm.bias"):
            errs[k[2:]] = rel(named[k[2:]].grad.double() - r["pre"][k[2:]].double(), v.grad)
    print(f"{name} end to end (normwise vs float64 autograd): " + " ".join(f"{k}={v:.2e}" for k, v in errs.items()))


C5 = dict(B=4, hw=(64, 64), L=300, lens=[300, 120, 1, 0])


def test_c5_block_as_benchmarked():
    t0 = time.time()
    r = _run(_block(False, torch.float32), **C5, ckpt=True, fp32_p=True, bucket=True)
    _check(r, "c5 fp32 master weights, fp32_attention, checkpointing, bucket views")
    r["rec"].trace.clear()                                           # the snapshots: room for the float64 autograd
    _end_to_end(r, "c5")
    print(f"case time {time.time() - t0:.1f} s")


def test_c5_block_bf16_params_autograd():
    t0 = time.time()
    r = _run(_block(False, torch.bfloat16), **C5, ckpt=False, fp32_p=False, bucket=False)
    _check(r, "c5 bf16 parameters, bf16 P, no checkpointing, autograd gradients")
    print(f"case time {time.time() - t0:.1f} s")


QK = dict(B=2, hw=(32, 32), L=300, lens=[300, 77])


def test_qk_norm_block_fp32_norm_weights():
    blk = _block(True, torch.float32)
    for j in "qk":                                                   # make sure the norm weights are off the bf16 grid
        w = getattr(blk.attn, j + "_norm").weight
        assert not torch.equal(w, w.to(torch.bfloat16).float())
    r = _run(blk, **QK, ckpt=True, fp32_p=True, bucket=True)
    _check(r, "qk_norm, fp32 norm weights")
    _end_to_end(r, "qk_norm")


def test_packed_block_forward_with_dropped_gates():
    """PixArtMSBlock.forward with packed captions (kv_off), B = 3 on a 24 x 40 grid, lens 300 / 77 / 9; sample 1's gate_msa
    and sample 2's gate_mlp are exactly 0, as drop path leaves them.  Their branch gradients (dy1, dy3) must be exact
    zeros (the stage check), while the gate gradients dm[2] / dm[5] of those samples stay non-zero."""
    r = _run(_block(False, torch.float32), B=3, hw=(24, 40), L=0, lens=[300, 77, 9], ckpt=True, fp32_p=True, bucket=False,
             packed=True, zero_gates=((1, 2), (2, 5)))
    assert (r["mod"][1, 2] == 0).all() and (r["mod"][2, 5] == 0).all()
    _check(r, "packed layout through PixArtMSBlock.forward, dropped gates")
    R, _ = _roles(r)
    N = r["N"]
    assert (R["dy1"][N:2 * N] == 0).all() and (R["dy3"][2 * N:] == 0).all()
    assert (R["dm2"][1] != 0).any() and (R["dm5"][2] != 0).any()
    _end_to_end(r, "packed")


@pytest.mark.parametrize("sampling,B,hw,ckpt", [("ave", 2, (15, 17), True), ("uniform", 2, (32, 32), False)])
def test_kv_compressed_block(sampling, B, hw, ckpt):
    """Parameter-free KV compression at scale factor 2: 'ave' on the odd 15 x 17 grid (7 x 8 kept keys), 'uniform' on
    32 x 32.  The kept k / v rows are picked in torch, and the backward scatters their gradients into the zero-filled
    dqkv; the references pick and scatter by the oracle's downsample_2d."""
    r = _run(_block(False, torch.float32, sampling=sampling), B=B, hw=hw, L=300, lens=[300, 57][:B], ckpt=ckpt, fp32_p=True,
             bucket=True)
    _check(r, f"KV compression {sampling} {hw[0]}x{hw[1]}")
    _end_to_end(r, f"KV compression {sampling}")


def _mutations(blk):
    def add_in_dropped(name, n, args, kw):
        if name == "ln_modulate_bwd" and n == 0:
            kw = {k: v for k, v in kw.items() if k != "add_in"}
        return args, kw

    def shift_scale_swapped(name, n, args, kw):
        if name == "ln_modulate" and n == 1:
            args[1], args[2] = args[2], args[1]
        return args, kw

    def fp32_norm_weight(name, n, args, kw):                         # the qk-norm backward before the fix
        if name == "ln_modulate_bwd" and n in (1, 2):
            w = (blk.attn.q_norm if n == 1 else blk.attn.k_norm).weight
            args[2] = (w.detach().float() - 1.0).view(1, C).contiguous()
        return args, kw

    return [("add_in dropped", "dx2 + dm[3,4]", add_in_dropped), ("shift / scale swapped", "xn2", shift_scale_swapped),
            ("fp32 norm weight in the qk-norm backward", "qk-norm backward", fp32_norm_weight)]


@pytest.mark.parametrize("which", [0, 1, 2])
def test_mutated_wiring_fails_at_its_stage(which):
    """Wrong data planted in one call of the real backward: the stage check must name that stage."""
    blk = _block(True, torch.float32)
    name, stage, fn = _mutations(blk)[which]
    r = _run(blk, **QK, ckpt=False, fp32_p=False, bucket=False, mutate=fn)
    st = bs.BlockStages(_inputs(r))
    with pytest.raises(bs.StageFailure) as e:
        st.run(_roles(r)[0])
    print(f"\nmutation '{name}': {str(e.value)[:300]}")
    for t in st.tallies.values():
        if t.bad:
            t.report()
    assert e.value.stage == stage
