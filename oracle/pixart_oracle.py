"""TEST INFRASTRUCTURE ONLY -- CPU restatement (the *oracle*) of the reference hot path
`PixArtMS.forward` -> 28 x `PixArtMSBlock.forward`.

Parity status: **pinned against the reference itself** -- the reference ships no tests or golden
vectors (SURVEY.md section 4), so this file is validated by `tests/test_oracle.py` against (a) the
unmodified reference model imported through `oracle/refshim.py` when `/root/reference` is present
(this container) and (b) the committed fixtures under `tests/golden/` that `oracle/gen_golden.py`
produced from that same reference (travels to the GPU box).

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may
import this module.  The product package `pixart_sigma_b200` never does: it has no CPU path.

Everything is functional: the model is a flat `state_dict` with the reference checkpoint key layout
(tools/convert_pixart_to_diffusers.py:30-155) plus an `OracleConfig`.  Math is done in `dtype`
(default fp32).  Each function cites the reference lines it follows (paths relative to
/root/reference/).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

Tensor = torch.Tensor


@dataclass
class OracleConfig:
    """Constructor arguments of PixArtMS (diffusion/model/nets/PixArtMS.py:91-112) that change the math."""
    input_size: int = 32
    patch_size: int = 2
    in_channels: int = 4
    hidden_size: int = 1152
    depth: int = 28
    num_heads: int = 16
    mlp_ratio: float = 4.0
    pred_sigma: bool = True
    pe_interpolation: float = 1.0
    model_max_length: int = 300
    micro_condition: bool = False
    qk_norm: bool = False
    kv_sampling: Optional[str] = None          # kv_compress_config['sampling']
    kv_scale_factor: int = 1                   # kv_compress_config['scale_factor']
    kv_compress_layer: Sequence[int] = field(default_factory=list)

    @property
    def out_channels(self) -> int:             # PixArt.py:90
        return self.in_channels * 2 if self.pred_sigma else self.in_channels

    @property
    def base_size(self) -> int:                # PixArt.py:100
        return self.input_size // self.patch_size

    def sr_ratio(self, layer: int) -> int:     # PixArtMS.py:155
        return int(self.kv_scale_factor) if layer in self.kv_compress_layer else 1


# ----------------------------------------------------------------------------- embeddings
def sincos_pos_embed(embed_dim: int, h: int, w: int, pe_interpolation: float, base_size: int) -> np.ndarray:
    """2-D sin/cos table, float64, shape (h*w, embed_dim).  Follows PixArt.py:258-307.

    Axis positions are arange(n)/(n/base_size)/pe_interpolation in float32; the *w* axis is the
    first meshgrid argument and feeds the first half of the channels (PixArt.py:267-270, 282-283).
    Each half is [sin(pos*omega), cos(pos*omega)] with omega_i = 10000^(-i/(D/4)) in float64 (:296-305).
    """
    assert embed_dim % 4 == 0
    pos_h = np.arange(h, dtype=np.float32) / (h / base_size) / pe_interpolation
    pos_w = np.arange(w, dtype=np.float32) / (w / base_size) / pe_interpolation
    gw, gh = np.meshgrid(pos_w, pos_h)                     # each (h, w): gw varies along columns
    quarter = embed_dim // 4
    omega = 1.0 / 10000 ** (np.arange(quarter, dtype=np.float64) / quarter)

    def axis_table(pos):                                   # (h*w,) -> (h*w, D/2)
        ang = pos.reshape(-1)[:, None] * omega[None, :]
        return np.concatenate([np.sin(ang), np.cos(ang)], axis=1)

    # Row-major flattening of the (h, w) grid matches the reference's reshape([2,1,w,h]) + reshape(-1):
    # the reshape only relabels dims, element order stays that of the (h, w) meshgrid.
    return np.concatenate([axis_table(gw), axis_table(gh)], axis=1)


def timestep_embedding(t: Tensor, dim: int = 256, max_period: float = 10000.0) -> Tensor:
    """fp32 sinusoid [cos | sin] of `t` (PixArt_blocks.py:282-299)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def _lin(sd: Dict[str, Tensor], name: str, x: Tensor) -> Tensor:
    return F.linear(x, sd[name + ".weight"], sd.get(name + ".bias"))


def timestep_mlp(sd, prefix: str, t: Tensor, dtype) -> Tensor:
    """TimestepEmbedder.forward (PixArt_blocks.py:301-304): sinusoid -> Linear -> SiLU -> Linear."""
    f = timestep_embedding(t, 256).to(dtype)
    return _lin(sd, prefix + ".mlp.2", F.silu(_lin(sd, prefix + ".mlp.0", f)))


def size_embed(sd, prefix: str, s: Tensor, bs: int, dtype) -> Tensor:
    """SizeEmbedder.forward (PixArt_blocks.py:328-339): every scalar of `s` gets its own embedding, concatenated."""
    if s.ndim == 1:
        s = s[:, None]
    if s.shape[0] != bs:
        s = s.repeat(bs // s.shape[0], 1)
    b, d = s.shape
    e = timestep_mlp(sd, prefix, s.reshape(-1), dtype)      # (b*d, outdim)
    return e.reshape(b, d * e.shape[-1])


def caption_embed(sd, y: Tensor) -> Tensor:
    """CaptionEmbedder eval path (PixArt_blocks.py:400-407): Mlp 4096 -> C (GELU tanh) -> C, no token drop."""
    h = F.gelu(_lin(sd, "y_embedder.y_proj.fc1", y), approximate="tanh")
    return _lin(sd, "y_embedder.y_proj.fc2", h)


# ----------------------------------------------------------------------------- block ops
def ln_modulate(x: Tensor, shift: Tensor, scale: Tensor, eps: float = 1e-6) -> Tensor:
    """LayerNorm(no affine, eps=1e-6) then x*(1+scale)+shift (PixArtMS.py:58,75; PixArt_blocks.py:24-25)."""
    return F.layer_norm(x, (x.shape[-1],), eps=eps) * (1 + scale) + shift


def sdpa_heads(q: Tensor, k: Tensor, v: Tensor) -> Tensor:
    """softmax(q k^T / sqrt(d)) v for (B, n, H, d) operands -- xformers default scale (PixArt_blocks.py:153)."""
    o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                       scale=q.shape[-1] ** -0.5)
    return o.transpose(1, 2)


def kv_downsample(sd, prefix: str, t: Tensor, H: int, W: int, sr: int, sampling: Optional[str]) -> Tensor:
    """AttentionKVCompress.downsample_2d (PixArt_blocks.py:97-121)."""
    if sampling is None or sr == 1:
        return t
    B, N, C = t.shape
    # the reference reshapes the [::sr] picks to int(N / sr) (int(H / sr) x int(W / sr)) tokens, which fails unless sr
    # divides the grid (:103, :107-108, :121)
    if sampling == "uniform_every":
        if N % sr:
            raise ValueError(f"'uniform_every' KV sampling needs the token count {N} to be a multiple of scale_factor {sr}")
        return t[:, ::sr]
    if sampling == "uniform" and (H % sr or W % sr):
        raise ValueError(f"'uniform' KV sampling needs scale_factor {sr} to divide the token grid {H} x {W}")
    img = t.reshape(B, H, W, C).permute(0, 3, 1, 2)
    if sampling == "ave":      # NB: the reference calls nearest-neighbour interpolation "ave" (:109-112)
        out = F.interpolate(img, scale_factor=1 / sr, mode="nearest").permute(0, 2, 3, 1)
    elif sampling == "uniform":
        out = img[:, :, ::sr, ::sr].permute(0, 2, 3, 1)
    elif sampling == "conv":   # depthwise conv k=s=sr (+bias) then LayerNorm(affine, eps 1e-5) (:84-89,115-117)
        out = F.conv2d(img, sd[prefix + ".sr.weight"], sd[prefix + ".sr.bias"], stride=sr, groups=C)
        out = out.reshape(B, C, -1).permute(0, 2, 1)
        out = F.layer_norm(out, (C,), sd[prefix + ".norm.weight"], sd[prefix + ".norm.bias"], eps=1e-5)
    else:
        raise ValueError(sampling)
    return out.reshape(B, -1, C)


def self_attention(sd, prefix: str, x: Tensor, HW: Tuple[int, int], heads: int, sr: int,
                   sampling: Optional[str], qk_norm: bool) -> Tensor:
    """AttentionKVCompress.forward (PixArt_blocks.py:123-158), mask=None as PixArtMSBlock calls it."""
    B, N, C = x.shape
    q, k, v = _lin(sd, prefix + ".qkv", x).reshape(B, N, 3, C).unbind(2)
    if qk_norm:                                              # :133-134, LayerNorm(dim) eps 1e-5 affine
        q = F.layer_norm(q, (C,), sd[prefix + ".q_norm.weight"], sd[prefix + ".q_norm.bias"])
        k = F.layer_norm(k, (C,), sd[prefix + ".k_norm.weight"], sd[prefix + ".k_norm.bias"])
    if sr > 1:
        k = kv_downsample(sd, prefix, k, HW[0], HW[1], sr, sampling)
        v = kv_downsample(sd, prefix, v, HW[0], HW[1], sr, sampling)
    d = C // heads
    o = sdpa_heads(q.reshape(B, N, heads, d), k.reshape(B, -1, heads, d), v.reshape(B, -1, heads, d))
    return _lin(sd, prefix + ".proj", o.reshape(B, N, C))


def cross_attention(sd, prefix: str, x: Tensor, cond: Tensor, y_lens: Sequence[int], heads: int) -> Tensor:
    """MultiHeadCrossAttention.forward (PixArt_blocks.py:43-58): packed keys, block-diagonal visibility.

    `cond` is (1, sum(y_lens), C); sample b's N queries see keys [off_b, off_b + y_lens[b]).
    """
    B, N, C = x.shape
    d = C // heads
    q = _lin(sd, prefix + ".q_linear", x).reshape(B, N, heads, d)
    kv = _lin(sd, prefix + ".kv_linear", cond).reshape(-1, 2, heads, d)
    outs, off = [], 0
    for b, L in enumerate(y_lens):
        L = int(L)
        if L == 0:                                           # empty key set -> zeros (xformers behaviour)
            outs.append(torch.zeros_like(q[b:b + 1]))
        else:
            outs.append(sdpa_heads(q[b:b + 1], kv[None, off:off + L, 0], kv[None, off:off + L, 1]))
        off += L
    return _lin(sd, prefix + ".proj", torch.cat(outs, 0).reshape(B, N, C))


def mlp(sd, prefix: str, x: Tensor) -> Tensor:
    """timm Mlp with GELU(tanh) (PixArtMS.py:66-67)."""
    return _lin(sd, prefix + ".fc2", F.gelu(_lin(sd, prefix + ".fc1", x), approximate="tanh"))


def block_forward(sd, prefix: str, x: Tensor, y: Tensor, t0: Tensor, y_lens: Sequence[int],
                  HW: Tuple[int, int], heads: int = 16, sr: int = 1, sampling: Optional[str] = None,
                  qk_norm: bool = False) -> Tensor:
    """PixArtMSBlock.forward (PixArtMS.py:71-79).  t0 is (B, 6*C); chunk order :74."""
    B, N, C = x.shape
    mod = sd[prefix + ".scale_shift_table"][None] + t0.reshape(B, 6, C)
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = mod.chunk(6, dim=1)
    x = x + gate_msa * self_attention(sd, prefix + ".attn", ln_modulate(x, shift_msa, scale_msa), HW,
                                      heads, sr, sampling, qk_norm)
    x = x + cross_attention(sd, prefix + ".cross_attn", x, y, y_lens, heads)
    x = x + gate_mlp * mlp(sd, prefix + ".mlp", ln_modulate(x, shift_mlp, scale_mlp))
    return x


def final_layer(sd, x: Tensor, t: Tensor) -> Tensor:
    """T2IFinalLayer.forward (PixArt_blocks.py:217-221) -- modulated by t, NOT t0."""
    shift, scale = (sd["final_layer.scale_shift_table"][None] + t[:, None]).chunk(2, dim=1)
    return _lin(sd, "final_layer.linear", ln_modulate(x, shift, scale))


def unpatchify(x: Tensor, h: int, w: int, p: int, c: int) -> Tensor:
    """(B, h*w, p*p*c) -> (B, c, h*p, w*p) (PixArtMS.py:236-248)."""
    B = x.shape[0]
    return x.reshape(B, h, w, p, p, c).permute(0, 5, 1, 3, 2, 4).reshape(B, c, h * p, w * p)


def pack_condition(y: Tensor, mask: Optional[Tensor]) -> Tuple[Tensor, List[int]]:
    """Mask packing of PixArtMS.forward (PixArtMS.py:196-204). y: (B,1,L,C) already embedded."""
    B, _, L, C = y.shape
    if mask is None:
        return y.squeeze(1).reshape(1, -1, C), [L] * B
    if mask.shape[0] != B:
        mask = mask.repeat(B // mask.shape[0], 1)
    mask = mask.squeeze(1).squeeze(1)
    packed = y.squeeze(1).masked_select(mask.unsqueeze(-1) != 0).view(1, -1, C)
    return packed, [int(v) for v in mask.sum(dim=1).tolist()]


# ----------------------------------------------------------------------------- whole model
@torch.no_grad()
def forward(sd: Dict[str, Tensor], cfg: OracleConfig, x: Tensor, timestep: Tensor, y: Tensor,
            mask: Optional[Tensor] = None, data_info: Optional[dict] = None,
            dtype: torch.dtype = torch.float32, return_intermediates: bool = False):
    """PixArtMS.forward (PixArtMS.py:165-211) in `dtype` on CPU.  Returns (B, out_channels, H, W)."""
    C, p = cfg.hidden_size, cfg.patch_size
    x, timestep, y = x.to(dtype), timestep.to(dtype), y.to(dtype)           # :173-175
    B = x.shape[0]
    h, w = x.shape[-2] // p, x.shape[-1] // p
    pos = torch.from_numpy(sincos_pos_embed(C, h, w, cfg.pe_interpolation, cfg.base_size)).unsqueeze(0).to(dtype)
    tok = F.conv2d(x, sd["x_embedder.proj.weight"], sd["x_embedder.proj.bias"], stride=p)
    tok = tok.flatten(2).transpose(1, 2) + pos                                # :184
    t = timestep_mlp(sd, "t_embedder", timestep, dtype)                       # :185
    if cfg.micro_condition:                                                   # :187-191
        csize = size_embed(sd, "csize_embedder", data_info["img_hw"].to(dtype), B, dtype)
        ar = size_embed(sd, "ar_embedder", data_info["aspect_ratio"].to(dtype), B, dtype)
        t = t + torch.cat([csize, ar], dim=1)
    t0 = _lin(sd, "t_block.1", F.silu(t))                                     # :193
    yp, y_lens = pack_condition(caption_embed(sd, y), mask)                   # :194-204
    inter = {"tokens": tok, "t": t, "t0": t0, "y_packed": yp, "y_lens": y_lens, "blocks": []}
    for i in range(cfg.depth):                                                # :205-206
        tok = block_forward(sd, f"blocks.{i}", tok, yp, t0, y_lens, (h, w), cfg.num_heads,
                            cfg.sr_ratio(i), cfg.kv_sampling, cfg.qk_norm)
        if return_intermediates:
            inter["blocks"].append(tok)
    out = unpatchify(final_layer(sd, tok, t), h, w, p, cfg.out_channels)      # :208-209
    return (out, inter) if return_intermediates else out


def forward_grad(sd, cfg, x, timestep, y, mask=None, data_info=None, dtype=torch.float32):
    """`forward` with autograd recording (the plain `forward` runs under no_grad): the fp32 reference for the
    training-backward parity tests -- gradients of this graph w.r.t. `sd` entries that require grad are what
    `loss.backward()` produces in the reference (train_scripts/train.py:197); pinned by tests/golden/train_*.pt."""
    return forward.__wrapped__(sd, cfg, x, timestep, y, mask=mask, data_info=data_info, dtype=dtype)


def forward_with_dpmsolver(sd, cfg, x, timestep, y, data_info=None, **kw) -> Tensor:
    """PixArtMS.forward_with_dpmsolver (PixArtMS.py:213-219): keep the eps half of the channels."""
    return forward(sd, cfg, x, timestep, y, data_info=data_info, **kw).chunk(2, dim=1)[0]


# ----------------------------------------------------------------------------- SDXL-VAE decoder ResBlock
def vae_resblock(sd: Dict[str, Tensor], prefix: str, x: Tensor, groups: int = 32, eps: float = 1e-6) -> Tensor:
    """diffusers ResnetBlock2D as used by the SDXL-VAE decoder (source not vendored in the reference;
    call site scripts/inference.py:136): GN32 -> SiLU -> conv3x3 -> GN32 -> SiLU -> conv3x3 (+1x1 shortcut)."""
    hdn = F.conv2d(F.silu(F.group_norm(x, groups, sd[prefix + ".norm1.weight"], sd[prefix + ".norm1.bias"], eps)),
                   sd[prefix + ".conv1.weight"], sd[prefix + ".conv1.bias"], padding=1)
    hdn = F.conv2d(F.silu(F.group_norm(hdn, groups, sd[prefix + ".norm2.weight"], sd[prefix + ".norm2.bias"], eps)),
                   sd[prefix + ".conv2.weight"], sd[prefix + ".conv2.bias"], padding=1)
    if prefix + ".conv_shortcut.weight" in sd:
        x = F.conv2d(x, sd[prefix + ".conv_shortcut.weight"], sd[prefix + ".conv_shortcut.bias"])
    return x + hdn


# ----------------------------------------------------------------------------- deterministic synthetic model
def state_dict_shapes(cfg: OracleConfig) -> Dict[str, Tuple[int, ...]]:
    """The checkpoint key/shape layout (SURVEY.md 8b; tools/convert_pixart_to_diffusers.py:30-155)."""
    C, p = cfg.hidden_size, cfg.patch_size
    Cm = int(C * cfg.mlp_ratio)
    s: Dict[str, Tuple[int, ...]] = {
        "x_embedder.proj.weight": (C, cfg.in_channels, p, p), "x_embedder.proj.bias": (C,),
        "t_embedder.mlp.0.weight": (C, 256), "t_embedder.mlp.0.bias": (C,),
        "t_embedder.mlp.2.weight": (C, C), "t_embedder.mlp.2.bias": (C,),
        "t_block.1.weight": (6 * C, C), "t_block.1.bias": (6 * C,),
        "y_embedder.y_proj.fc1.weight": (C, 4096), "y_embedder.y_proj.fc1.bias": (C,),
        "y_embedder.y_proj.fc2.weight": (C, C), "y_embedder.y_proj.fc2.bias": (C,),
        "y_embedder.y_embedding": (cfg.model_max_length, 4096),
        "final_layer.linear.weight": (p * p * cfg.out_channels, C), "final_layer.linear.bias": (p * p * cfg.out_channels,),
        "final_layer.scale_shift_table": (2, C),
    }
    if cfg.micro_condition:
        for e in ("csize_embedder", "ar_embedder"):
            s.update({f"{e}.mlp.0.weight": (C // 3, 256), f"{e}.mlp.0.bias": (C // 3,),
                      f"{e}.mlp.2.weight": (C // 3, C // 3), f"{e}.mlp.2.bias": (C // 3,)})
    for i in range(cfg.depth):
        b = f"blocks.{i}"
        s.update({
            f"{b}.scale_shift_table": (6, C),
            f"{b}.attn.qkv.weight": (3 * C, C), f"{b}.attn.qkv.bias": (3 * C,),
            f"{b}.attn.proj.weight": (C, C), f"{b}.attn.proj.bias": (C,),
            f"{b}.cross_attn.q_linear.weight": (C, C), f"{b}.cross_attn.q_linear.bias": (C,),
            f"{b}.cross_attn.kv_linear.weight": (2 * C, C), f"{b}.cross_attn.kv_linear.bias": (2 * C,),
            f"{b}.cross_attn.proj.weight": (C, C), f"{b}.cross_attn.proj.bias": (C,),
            f"{b}.mlp.fc1.weight": (Cm, C), f"{b}.mlp.fc1.bias": (Cm,),
            f"{b}.mlp.fc2.weight": (C, Cm), f"{b}.mlp.fc2.bias": (C,),
        })
        if cfg.sr_ratio(i) > 1 and cfg.kv_sampling == "conv":
            sr = cfg.sr_ratio(i)
            s.update({f"{b}.attn.sr.weight": (C, 1, sr, sr), f"{b}.attn.sr.bias": (C,),
                      f"{b}.attn.norm.weight": (C,), f"{b}.attn.norm.bias": (C,)})
        if cfg.qk_norm:
            for n in ("q_norm", "k_norm"):
                s.update({f"{b}.attn.{n}.weight": (C,), f"{b}.attn.{n}.bias": (C,)})
    return s


def synthetic_state_dict(cfg: OracleConfig, seed: int = 0, dtype=torch.float32) -> Dict[str, Tensor]:
    """Seeded random weights with *non-degenerate* values everywhere (the reference's own init zeroes
    cross_attn.proj and final_layer.linear, PixArtMS.py:279-285, which would make parity vacuous).
    Linear weights ~ N(0, 1/fan_in)-ish so activations stay O(1); used by GPU tests, smoke() and bench."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in state_dict_shapes(cfg).items():
        if k.endswith("scale_shift_table"):
            v = torch.randn(shp, generator=g) / cfg.hidden_size ** 0.5
        elif k.endswith("y_embedding"):
            v = torch.randn(shp, generator=g) / 4096 ** 0.5
        elif k.endswith("norm.weight") or k.endswith("_norm.weight"):
            v = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith(".sr.weight"):
            v = torch.full(shp, 1.0 / (shp[-1] * shp[-2])) + 0.05 * torch.randn(shp, generator=g)
        elif k.endswith(".bias"):
            v = 0.02 * torch.randn(shp, generator=g)
        else:
            fan_in = int(np.prod(shp[1:]))
            v = torch.randn(shp, generator=g) * (1.0 / fan_in) ** 0.5
        sd[k] = v.to(dtype)
    return sd


def rel_err(a: Tensor, b: Tensor) -> float:
    """Normwise relative error ||a-b||_2 / ||b||_2 (the parity metric, SURVEY.md Appendix D)."""
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def synthetic_inputs(cfg: OracleConfig, batch: int, latent_hw: Tuple[int, int], seed: int = 0,
                     timesteps: Optional[Sequence[float]] = None, lens: Optional[Sequence[int]] = None):
    """Seeded synthetic (x, timestep, y, mask) of SURVEY.md 8d: randn latents, randn T5 embeds
    (B,1,L,4096), fractional DPM-Solver timesteps, prefix masks of the given lengths (None -> no mask)."""
    g = torch.Generator().manual_seed(1000 + seed)
    H, W = latent_hw
    x = torch.randn(batch, cfg.in_channels, H, W, generator=g)
    y = torch.randn(batch, 1, cfg.model_max_length, 4096, generator=g)
    if timesteps is None:
        timesteps = [999.0 - 249.75 * (i % 4) for i in range(batch)]
    t = torch.tensor(list(timesteps), dtype=torch.float32)
    mask = None
    if lens is not None:
        mask = torch.zeros(batch, cfg.model_max_length, dtype=torch.long)
        for b, L in enumerate(lens):
            mask[b, :L] = 1
    return x, t, y, mask
