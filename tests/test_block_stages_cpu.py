"""The stage references of block_stages.py, on the CPU:

- Composition: chaining every stage's float64 reference on the outputs of the earlier ones (no rounding anywhere) gives
  float64 torch.autograd of `oracle.pixart_oracle.block_forward` -- x, mod, the caption rows and every parameter -- to
  ~1e-12.  This is the proof of the tests' own chain rule: with it, per-stage checks of the real kernels against these
  references leave no end-to-end tolerance to argue about.
- Teeth: kernel outputs emulated as each reference rounded once to its output dtype pass every stage; a wiring defect
  planted in one stage's output fails at that stage.

Block kinds: plain, qk_norm, and the parameter-free KV compressions 'uniform' and 'ave' (scale factor 2).  Geometry: C = 1152, 16 heads, a 4 x 6 token grid, B = 3 with the model's unpacked caption layout (L = 7 rows per sample,
kv_len 7, 3, 0: padding rows and an empty caption), sample 1's gate_msa = 0 (a sample drop path removed).
"""
import pytest
import torch

import block_stages as bs
from oracle import pixart_oracle as po

C, H, HW, LENS, L = 1152, 16, (4, 6), [7, 3, 0], 7
B, N = len(LENS), HW[0] * HW[1]
M = B * N
P = "blocks.0."


KINDS = {"plain": (False, None), "qk_norm": (True, None), "kv_uniform": (False, "uniform"), "kv_ave": (False, "ave")}
LN_EPS, QK_EPS = 1e-6, 1e-5          # the oracle's norm1 / norm2 and q_norm / k_norm


def _setup(kind, bf16):
    """(inputs of BlockStages, the oracle state dict, x, cond rows (B L, C), mod (B, 6, C), dout), float64.  bf16: weights,
    caption rows and dout hold bf16 values (as the kernels see them), x fp32 values."""
    qk_norm, sampling = KINDS[kind]
    cfg = po.OracleConfig(depth=1, qk_norm=qk_norm)
    sd = {k[len(P):]: v.double() for k, v in po.synthetic_state_dict(cfg, seed=3).items() if k.startswith(P)}
    g = torch.Generator().manual_seed(5)
    x = torch.randn(M, C, generator=g, dtype=torch.float64)
    cond = torch.randn(B * L, C, generator=g, dtype=torch.float64)
    mod = 0.3 * torch.randn(B, 6, C, generator=g, dtype=torch.float64)
    mod[1, 2] = 0.0                                               # gate_msa of sample 1: dropped
    dout = torch.randn(M, C, generator=g, dtype=torch.float64)
    w32 = {}
    if bf16:
        r = lambda t: t.to(torch.bfloat16).double()
        for k in sd:
            if k.endswith("norm.weight"):
                w32[k] = sd[k].float().double()                     # the fp32 master weight, off the bf16 grid
            sd[k] = r(sd[k])
        x, cond, dout = x.float().double(), r(cond), r(dout)
    inp = dict(x=x, cond=cond, mod=mod, dout=dout, B=B, N=N, H=H, keys=[(b * L, n) for b, n in enumerate(LENS)],
               W={t: sd[bs.MODULE[t] + ".weight"] for t in bs.TAGS}, bias={t: sd[bs.MODULE[t] + ".bias"] for t in bs.TAGS},
               qk={j: (sd[f"attn.{j}_norm.weight"], sd[f"attn.{j}_norm.bias"]) for j in "qk"} if qk_norm else None,
               qk_eps=QK_EPS, ln_eps=LN_EPS, kv_pick=(sampling, 2, HW) if sampling else None, fp32_p=False, splits=lambda m, n, k: bs.gb.auto_splits(m, n, k, 132),
               cast=(lambda t: t.to(torch.bfloat16).double()) if bf16 else (lambda t: t))
    inp["pre"] = {r_: torch.zeros_like(inp["W" if r_.startswith("dW") else "bias"][r_[3:]]) for r_ in
                  [f"d{k}.{t}" for t in bs.TAGS for k in "Wb"]}
    return inp, sd, w32


def _rel(a, b, scale=None):
    return ((a - b).norm() / (b.norm() if scale is None else scale)).item()


@pytest.mark.parametrize("kind", list(KINDS))
def test_stage_chain_composes_to_oracle_autograd(kind):
    qk_norm, sampling = KINDS[kind]
    inp, sd, _ = _setup(kind, bf16=False)
    R = {}
    bs.BlockStages(inp).run(R, emulate=bs.exact)
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    p["scale_shift_table"] = torch.zeros(6, C, dtype=torch.float64)             # mod = t0
    x = inp["x"].clone().view(B, N, C).requires_grad_(True)
    valid = torch.cat([torch.arange(b * L, b * L + n) for b, n in enumerate(LENS)])
    y = inp["cond"][valid].clone().requires_grad_(True)
    t0 = inp["mod"].clone().reshape(B, 6 * C).requires_grad_(True)
    out = po.block_forward({P + k: v for k, v in p.items()}, P[:-1], x, y[None], t0, LENS, HW, H, 2 if sampling else 1, sampling,
                           qk_norm)
    out.backward(inp["dout"].view(B, N, C))
    assert _rel(R["x3"], out.detach().reshape(M, C)) < 1e-12
    errs = {"x": _rel(R["dx"], x.grad.reshape(M, C)),
            "mod": _rel(torch.stack([R[f"dm{j}"] for j in range(6)], 1), t0.grad.view(B, 6, C)),
            "caption": _rel(R["dcond"][valid], y.grad)}
    assert (R["dcond"][~torch.isin(torch.arange(B * L), valid)] == 0).all(), "padding caption rows got a gradient"
    for t in bs.TAGS:
        errs[t + ".weight"] = _rel(R["dW." + t], p[bs.MODULE[t] + ".weight"].grad)
        errs[t + ".bias"] = _rel(R["db." + t], p[bs.MODULE[t] + ".bias"].grad)
    if qk_norm:
        for j in "qk":
            errs[f"{j}_norm.weight"] = _rel(R[f"dw.{j}_norm"].view(C), p[f"attn.{j}_norm.weight"].grad)
            # the k_norm bias moves every logit of a query alike: its exact gradient is 0 (rounding noise in both), so
            # its error is measured against the magnitude of the sum that forms it
            scale = R[f"d{j}1"].abs().sum(0).norm() if j == "k" else None
            errs[f"{j}_norm.bias"] = _rel(R[f"db.{j}_norm"].view(C), p[f"attn.{j}_norm.bias"].grad, scale)
    print(" ".join(f"{k}={v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) < 1e-12, errs


def _emulated(kind):
    inp, sd, w32 = _setup(kind, bf16=True)
    R = {}
    bs.BlockStages(inp).run(R, emulate=bs.round_to)
    return inp, R, w32


@pytest.mark.parametrize("kind", list(KINDS))
def test_rounded_emulation_passes_every_stage(kind):
    inp, R, _ = _emulated(kind)
    tallies = bs.BlockStages(inp).run(R)
    assert len(tallies) >= 40
    for t in tallies.values():
        t.report()
        assert t.ok()


def _defects():
    """(name, stage that must fail, block kind, function(inp, R, w32) planting the defect in R)."""
    rnd = bs.round_to
    b_of = torch.arange(M) // N

    def swapped_columns(inp, R, w32):
        ref, _ = bs._ln_fwd(inp["x"], inp["mod"][:, 1][b_of], inp["mod"][:, 0][b_of], LN_EPS)
        R["xn1"] = rnd(ref, torch.bfloat16)

    def add_in_dropped(inp, R, w32):
        R["dx2"] = rnd(R["dx2"] - inp["dout"], torch.float32)

    def dgate_rows(inp, R, w32):
        terms = inp["dout"] * R["y3"]
        R["dm5"] = rnd(bs._sample_sum(terms, torch.arange(M) // (N + 1), B), torch.float32)

    def fp32_norm_weight(inp, R, w32):
        w = w32["attn.q_norm.weight"]
        dx, _, _, _ = bs._ln_bwd(R["qkv"][:, :C], R["dq1"], (w - 1)[None].expand(M, C), 1e-5)
        R["dqn"] = rnd(dx, torch.float32)

    def dxb_not_added(inp, R, w32):
        R["dx1"] = R["dx2"].clone()

    def padding_key_gradient(inp, R, w32):
        R["dk2"] = R["dk2"].clone()
        R["dk2"][L + 3:2 * L] = 2.0 ** -20                         # rows past sample 1's 3 keys

    def unpicked_key_gradient(inp, R, w32):                       # dqkv not zero-filled where no kept key reads
        pick = bs.BlockStages(inp)._kv_rows(M)
        dk = torch.full((M, C), 2.0 ** -10, dtype=torch.float64)
        dv = torch.zeros(M, C, dtype=torch.float64)
        dk[pick], dv[pick] = R["dk1"].reshape(-1, C), R["dv1"].reshape(-1, C)
        R["dxn1"] = rnd(torch.cat([R["dq1"].reshape(M, C), dk, dv], 1) @ inp["W"]["qkv"], torch.bfloat16)

    def unguarded_gate(inp, R, w32):
        R["dy1"] = R["dy1"].clone()
        R["dy1"][N:2 * N] = rnd(R["dx1"][N:2 * N], torch.bfloat16)  # sample 1's gate is 0

    return [("shift and scale columns swapped", "xn1", "plain", swapped_columns),
            ("add_in dropped", "dx2 + dm[3,4]", "plain", add_in_dropped),
            ("dgate summed with the wrong rows_per_batch", "dy3 + dm[5]", "plain", dgate_rows),
            ("fp32 weight in the qk-norm backward", "qk-norm backward", "qk_norm", fp32_norm_weight),
            ("dxb not added into dx1", "dx1", "plain", dxb_not_added),
            ("padding key rows given a gradient", "cross-attention backward", "plain", padding_key_gradient),
            ("the unguarded gate of a dropped sample", "dy1 + dm[2]", "plain", unguarded_gate),
            ("unkept key rows of dqkv not zero-filled", "qkv", "kv_uniform", unpicked_key_gradient)]


@pytest.mark.parametrize("name,stage,kind,plant", _defects(), ids=[d[0] for d in _defects()])
def test_wiring_defect_fails_at_its_stage(name, stage, kind, plant):
    inp, R, w32 = _emulated(kind)
    plant(inp, R, w32)
    with pytest.raises(bs.StageFailure) as e:
        bs.BlockStages(inp).run(R)
    print(f"{name}: {e.value}")
    assert e.value.stage == stage, str(e.value)
