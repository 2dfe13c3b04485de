"""The head_dim-72 attention forward against a float64 reference, at the edges of its pipeline: key counts around the 128-key
block, key sets long enough that every K / V ring stage wraps its phase several times, query-tile tails, an empty key set between
full ones, and both P precisions with the lse output checked.

Bounds: the output normwise relative error per sample is held to 6e-3 with bf16 P (as the other attention tests) and to 3e-3
with bf16 hi + lo P (bf16 output rounding alone is about 1.2e-3); the log2-domain lse to 1e-5 relative (fp32 accumulation).
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from pixart_sigma_b200 import lib
DEV = "cuda"
D = 72
SENTINEL = -1280.0        # exactly representable in bf16 and fp32


def _ref(q, k, v, scale):
    """float64 softmax(q k^T scale) v and log2 sum exp2(q k^T scale log2 e) for (Nq, d) x (n, d) operands."""
    s = (q @ k.T) * scale
    lse = torch.logsumexp(s, -1)
    return torch.softmax(s, -1) @ v, lse / math.log(2.0)


def _run_and_check(lens, Nq, Nk, H, fp32_p, reverse, seed):
    B = len(lens)
    scale = D ** -0.5
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(B, Nq, H, D, generator=g) * 1.5).to(torch.bfloat16)
    k = torch.randn(B, Nk, H, D, generator=g).to(torch.bfloat16)
    v = torch.randn(B, Nk, H, D, generator=g).to(torch.bfloat16)
    ldo = H * D + 64
    obuf = torch.full((B * Nq, ldo), SENTINEL, dtype=torch.bfloat16, device=DEV)
    out = obuf[:, :H * D]
    lse = torch.full((B, H, Nq), SENTINEL, dtype=torch.float32, device=DEV)
    st = (H * D, D)
    lib.flash_attn(q.reshape(B * Nq, H * D).to(DEV), k.reshape(B * Nk, H * D).to(DEV), v.reshape(B * Nk, H * D).to(DEV), out,
                   B=B, H=H, Nq=Nq, Nk=Nk, kv_rows=B * Nk, kv_len=torch.tensor(lens, dtype=torch.int32, device=DEV),
                   q_strides=st, k_strides=st, v_strides=st, lse=lse, fp32_p=fp32_p, reverse_batch=reverse)
    torch.cuda.synchronize()
    got = obuf.double().cpu()
    assert (got[:, H * D:] == SENTINEL).all(), "the columns past H * 72 were written"
    got = got[:, :H * D].view(B, Nq, H, D)
    got_lse = lse.double().cpu()
    bound = 3e-3 if fp32_p else 6e-3
    for b, L in enumerate(lens):
        L = min(L, Nk)
        if L == 0:
            assert (got[b] == 0).all() and (got_lse[b] == 0).all(), f"sample {b}: no keys, so zero rows and lse 0"
            continue
        want = torch.empty(Nq, H, D, dtype=torch.float64)
        want_lse = torch.empty(H, Nq, dtype=torch.float64)
        for h in range(H):
            want[:, h], want_lse[h] = _ref(q[b, :, h].double(), k[b, :L, h].double(), v[b, :L, h].double(), scale)
        err = ((got[b] - want).norm() / want.norm()).item()
        lerr = ((got_lse[b] - want_lse).abs() / want_lse.abs().clamp(min=1)).max().item()
        assert err < bound, f"sample {b} ({L} keys): rel err {err:.2e}"
        assert lerr < 1e-5, f"sample {b} ({L} keys): lse rel err {lerr:.2e}"


@pytest.mark.parametrize("fp32_p", [False, True])
def test_key_counts_around_the_block(fp32_p):
    """1, 127, 128, 129, 255, 256, 257 keys side by side, an empty sample between full ones, a kv_len above Nk (clamped to Nk),
    and 200 queries (a full and a 72-row query tile)."""
    _run_and_check([1, 127, 128, 0, 129, 255, 256, 257, 400], Nq=200, Nk=257, H=2, fp32_p=fp32_p, reverse=False, seed=1)


@pytest.mark.parametrize("fp32_p", [False, True])
@pytest.mark.parametrize("reverse", [False, True])
def test_long_key_sets_wrap_the_ring(fp32_p, reverse):
    """3000 keys = 24 blocks, so each stage of the K and V rings is refilled 8 times and its barrier phase flips as often; the
    second sample ends in a partial block, and the third has no keys.  130 queries: a full tile and a 2-row tail."""
    _run_and_check([3000, 2900, 0], Nq=130, Nk=3000, H=3, fp32_p=fp32_p, reverse=reverse, seed=2)
