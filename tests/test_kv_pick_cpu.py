"""CPU tests of the parameter-free KV samplings (`model.kv_pick`, shared by the inference forward and the training
backward) against the reference's rule, AttentionKVCompress.downsample_2d (PixArt_blocks.py:97-121), and of the grids
the native paths reject.

'ave' is F.interpolate(scale_factor=1/sr, mode="nearest"): a floor(H/sr) x floor(W/sr) grid, not the ceil-sized
[::sr, ::sr] pick.  The two differ whenever sr does not divide a side, e.g. on the 15 x 17 and 9 x 27 token grids of
non-square aspect buckets."""
import pytest
import torch
import torch.nn.functional as F

from oracle import pixart_oracle as po
from pixart_sigma_b200 import autograd as ag
from pixart_sigma_b200.model import AttentionKVCompress, PixArtMSBlock, check_kv_conv_grid, kv_pick


def _grid_ids(B, H, W):
    """(B*H*W, 1) float tensor whose value is the row index: a pick of it reads back which tokens were kept."""
    return torch.arange(B * H * W, dtype=torch.float32).view(B * H * W, 1)


@pytest.mark.parametrize("sr", [2, 3, 4])
def test_ave_pick_selects_what_nearest_interpolation_selects(sr):
    """Over H, W in 1..40: the kept token indices equal those F.interpolate(scale_factor=1/sr, mode="nearest") selects;
    where interpolation has no output (a side shorter than sr) the pick raises ValueError."""
    B = 2
    for H in range(1, 41):
        for W in range(1, 41):
            t = _grid_ids(B, H, W)
            img = t.view(B, H, W, 1).permute(0, 3, 1, 2)
            try:
                want = F.interpolate(img, scale_factor=1 / sr, mode="nearest").permute(0, 2, 3, 1)
            except RuntimeError:
                with pytest.raises(ValueError):
                    kv_pick(t, B, (H, W), "ave", sr)
                continue
            got = kv_pick(t, B, (H, W), "ave", sr)
            assert got.shape == want.shape == (B, H // sr, W // sr, 1), (H, W, sr)
            assert torch.equal(got, want), (H, W, sr)


def test_ave_pick_on_odd_grids_keeps_the_floor_sized_grid():
    t = _grid_ids(1, 15, 17)
    assert kv_pick(t, 1, (15, 17), "ave", 2).shape == (1, 7, 8, 1)
    assert kv_pick(_grid_ids(1, 9, 27), 1, (9, 27), "ave", 2).shape == (1, 4, 13, 1)
    assert kv_pick(_grid_ids(1, 16, 16), 1, (16, 16), "ave", 3).shape == (1, 5, 5, 1)


@pytest.mark.parametrize("sr", [2, 3, 4])
def test_uniform_picks_follow_the_reference_or_raise(sr):
    """'uniform' is the [::sr, ::sr] pick where sr divides H and W and raises ValueError elsewhere (the reference's reshape
    to int(H/sr) x int(W/sr) tokens fails there); 'uniform_every' likewise over the N = H W tokens.  The oracle's
    kv_downsample follows the same rule."""
    B, C = 2, 3
    for H in range(1, 21):
        for W in range(1, 21):
            t = torch.randn(B * H * W, C)
            if H % sr or W % sr:
                with pytest.raises(ValueError):
                    kv_pick(t, B, (H, W), "uniform", sr)
                with pytest.raises(ValueError):
                    po.kv_downsample({}, "", t.view(B, H * W, C), H, W, sr, "uniform")
            else:
                want = t.view(B, H, W, C)[:, ::sr, ::sr]
                assert torch.equal(kv_pick(t, B, (H, W), "uniform", sr), want)
                assert torch.equal(po.kv_downsample({}, "", t.view(B, H * W, C), H, W, sr, "uniform"), want.reshape(B, -1, C))
            if (H * W) % sr:
                with pytest.raises(ValueError):
                    kv_pick(t, B, (H, W), "uniform_every", sr)
                with pytest.raises(ValueError):
                    po.kv_downsample({}, "", t.view(B, H * W, C), H, W, sr, "uniform_every")
            else:
                want = t.view(B, H * W, C)[:, ::sr]
                assert torch.equal(kv_pick(t, B, (H, W), "uniform_every", sr), want)
                assert torch.equal(po.kv_downsample({}, "", t.view(B, H * W, C), H, W, sr, "uniform_every"), want)


def test_kv_pick_is_a_view_the_backward_can_scatter_into():
    """The training backward copies the compressed-key gradients into the pick of the dk slice of dqkv: the pick must be
    a view of that slice, and a scatter through it must leave every other element alone."""
    B, H, W, C = 2, 15, 17, 4
    dqkv = torch.zeros(B * H * W, 3 * C)
    dk = dqkv[:, C:2 * C]
    pick = kv_pick(dk, B, (H, W), "ave", 2)
    assert pick.data_ptr() == dk.data_ptr()
    pick.copy_(torch.ones(pick.shape))
    want = torch.zeros(B, H, W, 3 * C)
    want[:, 0:14:2, 0:16:2, C:2 * C] = 1
    assert torch.equal(dqkv.view(B, H, W, 3 * C), want)


def _attn(sampling, sr, C=16):
    return AttentionKVCompress(C, num_heads=1, sampling=sampling, sr_ratio=sr)


@pytest.mark.parametrize("HW", [(15, 17), (9, 27), (16, 15)])
def test_native_paths_reject_grids_the_reference_cannot_take(HW):
    """'uniform' with sr not dividing the grid raises ValueError, and 'conv' on an odd grid (the fused kernel needs even
    H, W) raises NotImplementedError, in the training and the inference path, before any kernel is called (these run
    on the CPU, where a kernel call would fail differently)."""
    B, C = 2, 16
    N = HW[0] * HW[1]
    qkv = torch.zeros(B * N, 3 * C, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="divide the token grid"):
        ag._compress_kv(_attn("uniform", 2, C), qkv, B, N, HW)
    with pytest.raises(NotImplementedError, match="even token grid"):
        ag._compress_kv(_attn("conv", 2, C), qkv, B, N, HW)
    if N % 2:
        with pytest.raises(ValueError, match="multiple of scale_factor"):
            ag._compress_kv(_attn("uniform_every", 2, C), qkv, B, N, HW)
    for sampling, err in (("uniform", ValueError), ("conv", NotImplementedError)):
        blk = PixArtMSBlock(C, 1, sampling=sampling, sr_ratio=2)
        with pytest.raises(err):
            blk._compress_kv(qkv, B, N, HW, blk._ws)
    with pytest.raises(NotImplementedError, match="scale_factor 2"):
        check_kv_conv_grid((16, 16), 3)
    check_kv_conv_grid((16, 24), 2)
