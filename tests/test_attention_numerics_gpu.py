"""Element-wise float64 contracts of the attention kernels on real softmax distributions (-m gpu): lib.flash_attn (bf16 P
and bf16 hi + lo P), lib.flash_attn_bwd and lib.t5_attn against attn_bounds.py, whose slack is derived from the kernels'
arithmetic (see its docstring; test_attention_numerics_cpu.py checks it against an emulation of that arithmetic).

Every output element must lie within ulp(ref) + slack of the float64 reference, and the bias statistic
mean(sign(ref) (got - ref) / bound) must stay within attn_bounds.MAX_BIAS: rounding P or dS toward zero passes the worst-case
bound but not that.  The distributions are those of attn_bounds.make_inputs (diffuse, peaked in both key orders, logits
offset by ~200 log2 units, values and keys offset).  The geometries: self-attention at 256, 1024 and 4096 tokens (H = 16,
B = 2; 4096 is the 1024-px step, with more CTAs than SMs), the odd token grids 15 x 17 and 9 x 27, KV-compressed keys (4096
x 1024, and the 56 keys 'ave' keeps of a 15 x 17 grid at sr 2), and packed cross-attention with kv_off, captions of 300,
77, 1 and 120 tokens, an empty sample and a kv_len above Nk.  Inputs are read through a head stride of 80 whose padding is
NaN; the forward writes into a sentinel-banded buffer; the backward writes the interleaved (rows, 3, H, 72) buffer of
self-attention, or the packed (rows, 2, H, 72) cross keys, where rows at or past kv_len must stay untouched.  The references
are computed in float64 on the GPU, one (sample, head) at a time.  With -s every output prints its largest error / bound,
the fraction of elements correctly rounded and the bias.
"""
import pytest
import torch

import attn_bounds as ab
from test_numerics_gpu import SENTINEL, _assert_pad_unchanged, _padded

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
DEV = "cuda"
D, HS = 72, 80
SCALE = D ** -0.5
NAN = float("nan")

# (id, layout, B, H, Nq, Nk, key lengths or None, distributions)
GEOMETRIES = [
    ("self256", "self", 2, 16, 256, 256, None, ["diffuse", "offset_vk"]),
    ("self1024", "self", 2, 16, 1024, 1024, None, ab.DISTRIBUTIONS),
    ("self4096", "self", 2, 16, 4096, 4096, None, ["diffuse", "peaked", "offset_vk"]),
    ("grid15x17", "self", 3, 16, 255, 255, None, ["diffuse", "peaked"]),
    ("grid9x27", "self", 3, 16, 243, 243, None, ["diffuse", "offset_logits"]),
    ("kv4096x1024", "kv", 2, 16, 4096, 1024, None, ["diffuse", "offset_vk"]),
    ("ave15x17", "kv", 3, 16, 255, 56, None, ["diffuse", "peaked_rev"]),
    ("cross", "packed", 5, 16, 256, 256, [300, 77, 1, 0, 120], ["diffuse", "offset_vk"]),
]
CASES = [pytest.param(lay, B, H, Nq, Nk, lens, dist, id=f"{gid}-{dist}")
         for gid, lay, B, H, Nq, Nk, lens, dists in GEOMETRIES for dist in dists]


def _heads(x):
    """(B, H, N, D) float64 -> (B N, H, D) bf16 on the device."""
    return x.permute(0, 2, 1, 3).reshape(-1, x.shape[1], D).to(torch.bfloat16)


@pytest.mark.parametrize("layout,B,H,Nq,Nk,lens,dist", CASES)
def test_flash_attn_forward_and_backward_elementwise(layout, B, H, Nq, Nk, lens, dist):
    C = H * D
    lens = lens or [Nk] * B
    eff = [min(L_, Nk) for L_ in lens]                       # the kernels attend to min(kv_len, Nk) keys
    Lmax = max(lens)
    q, k, v, do = ab.make_inputs(dist, (B, H), Nq, Lmax, D, seed=Nq + 7 * Nk + B, device=DEV)
    if layout == "self":                                      # the (B N, 3, H, 80) qkv buffer, padding NaN
        buf = torch.full((B * Nq, 3, H, HS), NAN, dtype=torch.bfloat16, device=DEV)
        for i, x in enumerate((q, k, v)):
            buf[:, i, :, :D] = _heads(x)
        qv, kv_, vv = buf[:, 0], buf[:, 1], buf[:, 2]
        qs = ks = (3 * H * HS, HS)
        kv_rows, offs, kv_len, kv_off = B * Nk, [b * Nk for b in range(B)], None, None
    else:
        qb = torch.full((B * Nq, H, HS), NAN, dtype=torch.bfloat16, device=DEV)
        qb[:, :, :D] = _heads(q)
        qv, qs = qb, (H * HS, HS)
        offs = [sum(lens[:b]) for b in range(B)] if layout == "packed" else [b * Nk for b in range(B)]
        kv_rows = sum(lens) if layout == "packed" else B * Nk
        kb = torch.full((kv_rows, 2, H, HS), NAN, dtype=torch.bfloat16, device=DEV)
        for b, L_ in enumerate(lens):
            kb[offs[b]:offs[b] + L_, 0, :, :D] = _heads(k[b:b + 1, :, :L_])
            kb[offs[b]:offs[b] + L_, 1, :, :D] = _heads(v[b:b + 1, :, :L_])
        kv_, vv = kb[:, 0], kb[:, 1]
        ks = (2 * H * HS, HS)
        kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV) if layout == "packed" else None
        kv_off = torch.tensor(offs, dtype=torch.int32, device=DEV) if layout == "packed" else None
    geo = dict(B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=kv_rows, kv_len=kv_len, kv_off=kv_off, q_strides=qs, k_strides=ks,
               v_strides=ks, scale=SCALE)
    outs = {}
    for split in (False, True):
        out, obuf = _padded(B * Nq, C, 64, SENTINEL, torch.bfloat16)
        before = obuf.clone()
        lse = torch.full((B, H, Nq), NAN, dtype=torch.float32, device=DEV)
        lib.flash_attn(qv, kv_, vv, out, lse=lse, fp32_p=split, **geo)
        torch.cuda.synchronize()
        _assert_pad_unchanged(obuf, C, before, "out")
        outs[split] = (out, lse)
    out, lse = outs[False]

    dod, _ = _padded(B * Nq, C, 64, NAN, torch.bfloat16)
    dod.copy_(_heads(do).reshape(B * Nq, C))
    if layout == "self":
        dqkv = torch.full((B * Nq, 3, H, D), SENTINEL, dtype=torch.bfloat16, device=DEV)
        dq, dk, dv = dqkv[:, 0], dqkv[:, 1], dqkv[:, 2]
        dqs = dks = (3 * C, D)
        bands = []
    else:
        dq, dqbuf = _padded(B * Nq, C, 64, SENTINEL, torch.bfloat16)
        dkv, dkvbuf = _padded(kv_rows, 2 * C, 64, SENTINEL, torch.bfloat16)
        dk, dv = dkv[:, :C], dkv[:, C:]
        dqs, dks = (dq.stride(0), D), (dkv.stride(0), D)
        bands = [(dqbuf, C, dqbuf.clone()), (dkvbuf, 2 * C, dkvbuf.clone())]
    lib.flash_attn_bwd(qv, kv_, vv, out, dod, lse, dq, dk, dv, dq_strides=dqs, dk_strides=dks, dv_strides=dks, **geo)
    torch.cuda.synchronize()
    for buf, cols, bb in bands:
        _assert_pad_unchanged(buf, cols, bb, "gradient buffer")

    names = ("o", "o_hi_lo", "lse", "dq", "dk", "dv")
    tal = {n_: ab.Tally(f"{dist} {n_}", fp32=(n_ == "lse")) for n_ in names}
    got_o = {s_: outs[s_][0].view(B, Nq, H, D) for s_ in outs}
    got_lse = {s_: outs[s_][1].double() for s_ in outs}
    gq = dq.reshape(B, Nq, H, D) if layout != "self" else dqkv[:, 0].view(B, Nq, H, D)
    dk3, dv3 = dk.view(-1, H, D) if layout == "self" else dk.reshape(-1, H, D), dv.reshape(-1, H, D)
    for b, L_ in enumerate(eff):
        rows = slice(offs[b], offs[b] + L_)
        if L_ == 0:                                           # no keys: zero output, lse 0, zero dQ
            for s_ in outs:
                assert (got_o[s_][b] == 0).all() and (got_lse[s_][b] == 0).all(), f"empty sample {b}"
            assert (gq[b] == 0).all(), f"dQ of the empty sample {b}"
            continue
        if layout != "self":                                  # dK / dV rows at or past kv_len: untouched
            past = slice(offs[b] + L_, offs[b] + lens[b])
            assert (dk3[past] == SENTINEL).all() and (dv3[past] == SENTINEL).all(), f"dK / dV past kv_len, sample {b}"
        for h in range(H):
            qh, kh, vh, doh = q[b, h], k[b, h, :L_], v[b, h, :L_], do[b, h]
            fw = ab.forward(qh, kh, vh, SCALE)
            tal["o"].add(got_o[False][b, :, h], fw["o"], fw["slack_o"])
            tal["lse"].add(got_lse[False][b, h], fw["lse"], fw["slack_lse"])
            tal["lse"].add(got_lse[True][b, h], fw["lse"], fw["slack_lse"])
            fs = ab.forward(qh, kh, vh, SCALE, split_p=True)
            tal["o_hi_lo"].add(got_o[True][b, :, h], fs["o"], fs["slack_o"])
            bw = ab.backward(qh, kh, vh, doh, got_o[False][b, :, h].double(), got_lse[False][b, h], SCALE, fwd=fw)
            tal["dq"].add(gq[b, :, h], bw["dq"], bw["slack_dq"])
            tal["dk"].add(dk3[rows, h], bw["dk"], bw["slack_dk"])
            tal["dv"].add(dv3[rows, h], bw["dv"], bw["slack_dv"])
            del fw, fs, bw
    if layout == "self":
        assert not (dqkv == SENTINEL).any(), "a gradient element was not written"
    for t in tal.values():
        t.check()


T5_CASES = [pytest.param(B, H, L, lens, dense, id=f"B{B}H{H}L{L}-{'dense' if dense else 'toeplitz'}")
            for B, H, L, lens in [(2, 64, 300, [300, 77]), (3, 4, 130, [130, 64, 1])] for dense in (True, False)]


@pytest.mark.parametrize("B,H,L,lens,dense", T5_CASES)
def test_t5_attn_elementwise(B, H, L, lens, dense):
    """lib.t5_attn (head_dim 64, scale 1, 64-key blocks) against the same forward contract with the bias joining the logit
    error (attn_bounds: 3u log2(e) |bias|, u |t| for the separate product).  T5 logits are unscaled: N(0, 1) q and k give
    logits of standard deviation 8, the peaked case, plus a relative-position bias of standard deviation 3 ([H, L, L] or the
    Toeplitz [H, 2L - 1] form) and finfo.min key masks past each caption's length; out is a slice of a sentinel-banded
    buffer."""
    Dt = 64
    g = torch.Generator(device=DEV).manual_seed(L + H)
    n = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64, device=DEV)
    q, k, v = (n(B, H, L, Dt).to(torch.bfloat16).double() for _ in range(3))
    rel = (n(H, 2 * L - 1) * 3).float()
    i = torch.arange(L, device=DEV)
    bias = rel[:, (i[None, :] - i[:, None]) + L - 1].contiguous()     # bias[h, i, j] = rel[h, j - i + L - 1]
    key_bias = torch.zeros(B, L, dtype=torch.float32, device=DEV)
    for b, Lb in enumerate(lens):
        key_bias[b, Lb:] = torch.finfo(torch.float32).min
    rows = lambda x: x.permute(0, 2, 1, 3).reshape(B * L, H * Dt).to(torch.bfloat16)
    out, obuf = _padded(B * L, H * Dt, 64, SENTINEL, torch.bfloat16)
    before = obuf.clone()
    lib.t5_attn(rows(q), rows(k), rows(v), out, bias if dense else None, key_bias, B=B, H=H, L=L, scale=1.0,
                rel_bias=None if dense else rel)
    torch.cuda.synchronize()
    _assert_pad_unchanged(obuf, H * Dt, before, "t5 out")
    got = out.view(B, L, H, Dt)
    tal = ab.Tally("t5 o")
    for b in range(B):
        for h in range(H):
            fw = ab.forward(q[b, h], k[b, h], v[b, h], 1.0, blk=64, bias=bias[h].double() + key_bias[b].double())
            tal.add(got[b, :, h], fw["o"], fw["slack_o"])
    tal.check()
