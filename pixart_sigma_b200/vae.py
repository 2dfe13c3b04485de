"""SDXL-VAE decoder ResBlock on the sm_90a implicit-GEMM 3x3 convolution (SURVEY.md 8a row 19).

The reference decodes latents with diffusers' `AutoencoderKL` (scripts/inference.py:136, 193-196); diffusers is not
vendored in the reference and not installed here, so this module mirrors the public `ResnetBlock2D` of the SDXL-VAE
decoder -- parameter names `norm1, conv1, norm2, conv2, conv_shortcut`, GroupNorm(32, eps 1e-6) -> SiLU -> Conv3x3 twice,
1x1 shortcut when the channel count changes -- with both 3x3 convolutions (68 % of the decoder FLOPs) on
`pxa_conv3x3_nhwc_bf16` and GroupNorm + SiLU in front of each as one NHWC kernel pair (`pxa_groupnorm_silu_nhwc_bf16`:
statistics, apply), so a block is 2 convolutions + 2 x 2 light passes with no layout copies in between.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import lib


class DecoderResBlock(nn.Module):
    def __init__(self, in_channels: int, out_channels: Optional[int] = None, groups: int = 32, eps: float = 1e-6):
        super().__init__()
        out_channels = out_channels or in_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None
        self._packed = {}

    def _pack(self, conv: nn.Conv2d) -> torch.Tensor:
        """[Cout, Cin, 3, 3] -> [Cout, 3, 3, Cin] (tap-major K), cached until the parameter changes."""
        key = (id(conv), conv.weight._version, conv.weight.data_ptr())
        hit = self._packed.get(id(conv))
        if hit is None or hit[0] != key:
            hit = (key, conv.weight.detach().permute(0, 2, 3, 1).contiguous())
            self._packed[id(conv)] = hit
        return hit[1]

    @torch.no_grad()
    def forward(self, x: torch.Tensor, temb=None) -> torch.Tensor:
        """x (B, C, H, W) bf16 on a H100 -> (B, Cout, H, W) bf16 (channels_last memory format)."""
        _need_kernels(x, self.conv1.weight, "DecoderResBlock")
        B, Cc, H, W = x.shape
        x = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)     # no copy when the caller already is NHWC
        x_nhwc = x.permute(0, 2, 3, 1)                                          # contiguous (B, H, W, C) view
        h = lib.groupnorm_silu_nhwc(x_nhwc, self.norm1.weight, self.norm1.bias, torch.empty_like(x_nhwc),
                                    groups=self.norm1.num_groups, eps=self.norm1.eps)
        h1 = torch.empty(B, H, W, self.out_channels, dtype=torch.bfloat16, device=x.device)
        lib.conv3x3_nhwc(h, self._pack(self.conv1), self.conv1.bias, h1)
        h2 = lib.groupnorm_silu_nhwc(h1, self.norm2.weight, self.norm2.bias, torch.empty_like(h1),
                                     groups=self.norm2.num_groups, eps=self.norm2.eps)
        if self.conv_shortcut is not None:
            sc = torch.empty(B * H * W, self.out_channels, dtype=torch.bfloat16, device=x.device)
            lib.gemm(x_nhwc.reshape(B * H * W, Cc), self.conv_shortcut.weight.view(self.out_channels, Cc),
                     self.conv_shortcut.bias, sc)
            sc = sc.view(B, H, W, self.out_channels)
        else:
            sc = x_nhwc
        out = torch.empty(B, H, W, self.out_channels, dtype=torch.bfloat16, device=x.device)
        lib.conv3x3_nhwc(h2, self._pack(self.conv2), self.conv2.bias, out, residual=sc.contiguous())
        return out.permute(0, 3, 1, 2)


class UpsampleConv(nn.Module):
    """Nearest-neighbour x2 upsample followed by a 3x3 convolution (diffusers `Upsample2D` of the SDXL-VAE decoder up
    blocks; 2.8 TFLOP of the 10.5 TFLOP decode at 1024px).  The interpolation is data movement (PyTorch); the
    convolution runs on `pxa_conv3x3_nhwc_bf16`."""

    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)
        self._packed = None

    @torch.no_grad()
    def forward(self, x: torch.Tensor, *args, **kwargs) -> torch.Tensor:
        _need_kernels(x, self.conv.weight, "UpsampleConv")
        key = (self.conv.weight._version, self.conv.weight.data_ptr())
        if self._packed is None or self._packed[0] != key:
            self._packed = (key, self.conv.weight.detach().permute(0, 2, 3, 1).contiguous())
        B, Cc, H, W = x.shape
        up = F.interpolate(x.to(torch.bfloat16), scale_factor=2.0, mode="nearest")
        up = up.contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)           # (B, 2H, 2W, C)
        out = torch.empty(B, 2 * H, 2 * W, Cc, dtype=torch.bfloat16, device=x.device)
        lib.conv3x3_nhwc(up, self._packed[1], self.conv.bias, out)
        return out.permute(0, 3, 1, 2)


def patch_diffusers_decoder(vae) -> int:
    """Route every ResnetBlock2D of a diffusers AutoencoderKL *decoder* through `DecoderResBlock` (shares the
    parameters).  Returns the number of blocks patched.  (diffusers is not installed in the build container; this is
    the binding a user of scripts/inference.py adds after loading `vae`.)"""
    n = 0
    for mod in vae.decoder.modules():
        if type(mod).__name__ == "ResnetBlock2D" and getattr(mod, "time_emb_proj", None) is None:
            blk = DecoderResBlock(mod.in_channels, mod.out_channels, mod.norm1.num_groups, mod.norm1.eps)
            blk.norm1, blk.conv1, blk.norm2, blk.conv2 = mod.norm1, mod.conv1, mod.norm2, mod.conv2
            blk.conv_shortcut = getattr(mod, "conv_shortcut", None)
            scale = getattr(mod, "output_scale_factor", 1.0)
            mod.forward = (lambda b, s: (lambda x, temb=None, *a, **k: b(x) / s))(blk, scale)
            n += 1
        elif type(mod).__name__ == "Upsample2D" and getattr(mod, "conv", None) is not None and mod.conv.kernel_size == (3, 3):
            up = UpsampleConv(mod.conv.in_channels)
            up.conv = mod.conv
            mod.forward = (lambda u: (lambda x, *a, **k: u(x)))(up)
            n += 1
    return n


# ------------------------------------------------------------------------------------------------- the whole autoencoder
# SURVEY.md 8(f).2: the rest of the SDXL-VAE around the ResBlock convolutions.  Module / parameter names follow diffusers'
# AutoencoderKL (`decoder.conv_in`, `decoder.mid_block.resnets.0`, `decoder.mid_block.attentions.0.{group_norm,to_q,to_k,to_v,
# to_out.0}`, `decoder.up_blocks.i.resnets.j`, `decoder.up_blocks.i.upsamplers.0.conv`, `decoder.conv_norm_out`,
# `decoder.conv_out`, `post_quant_conv`; `encoder.*` / `quant_conv` alike), so the `vae/diffusion_pytorch_model.safetensors` of
# `PixArt-alpha/pixart_sigma_sdxlvae_T5_diffusers` loads with `load_state_dict` (call sites scripts/inference.py:136,193-196 and
# train_scripts/train.py:85-88,149).  Every 3x3 convolution with >= 64 input channels (99.8 % of the decoder FLOPs) runs on
# `pxa_conv3x3_nhwc_bf16`, every GroupNorm (+SiLU) on `pxa_groupnorm_silu_nhwc_bf16`, the 1x1 / Linear layers on `pxa_gemm_bf16`;
# activations stay NHWC bf16 from conv_in to conv_out.  What stays PyTorch (north_star: "SDXL-VAE stay[s] PyTorch except the decoder
# ResBlock convs"): conv_in (4 channels in), conv_out (3 channels out), the stride-2 down-sampling convolutions of the encoder, the
# 4 / 8-channel 1x1 quant convolutions, and the softmax(QK^T)V of the single-head mid-block attention (head_dim 512).
SDXL_VAE_CONFIG = dict(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                       norm_num_groups=32, scaling_factor=0.13025)


def _need_kernels(t: torch.Tensor, w: torch.Tensor, what: str):
    if not t.is_cuda or w.dtype != torch.bfloat16:
        raise RuntimeError(f"{what} runs on the sm_90a kernels only: CUDA tensors and bf16 weights required")


def _nhwc(x: torch.Tensor) -> torch.Tensor:
    """(B, C, H, W) any layout -> contiguous (B, H, W, C) bf16 view (no copy when x is already channels_last bf16)."""
    return x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)


def _conv3x3(conv: nn.Conv2d, x_nhwc: torch.Tensor, cache: dict) -> torch.Tensor:
    """3x3 / stride 1 / pad 1 convolution of an NHWC bf16 image with a checkpoint-layout `nn.Conv2d`; NHWC out.  `cache` keeps the
    tap-major copy of the weight until the parameter changes."""
    if conv.in_channels % 64 or conv.out_channels % 8:              # conv_in / conv_out: 4 in / 3 out channels (PyTorch, see above)
        y = F.conv2d(x_nhwc.permute(0, 3, 1, 2), conv.weight, conv.bias, padding=1)
        return y.contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)
    key = (conv.weight._version, conv.weight.data_ptr())
    if cache.get("key") != key:
        cache["key"], cache["w"] = key, conv.weight.detach().permute(0, 2, 3, 1).contiguous()
    B, H, W, _ = x_nhwc.shape
    out = torch.empty(B, H, W, conv.out_channels, dtype=torch.bfloat16, device=x_nhwc.device)
    return lib.conv3x3_nhwc(x_nhwc.contiguous(), cache["w"], conv.bias, out)


class MidBlockAttention(nn.Module):
    """diffusers `Attention(512, heads=1, dim_head=512, norm_num_groups=32, eps=1e-6, residual_connection=True, bias=True)`
    of the VAE mid block: GroupNorm -> q / k / v Linear -> softmax(q k^T / sqrt(512)) v over the H*W positions -> Linear -> + x.
    GroupNorm and the four Linear layers (q, k, v as ONE GEMM over the row-stacked weights) run on the kernels."""

    def __init__(self, channels: int, groups: int = 32, eps: float = 1e-6):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, channels, eps=eps)
        self.to_q, self.to_k, self.to_v = (nn.Linear(channels, channels) for _ in range(3))
        self.to_out = nn.ModuleList([nn.Linear(channels, channels), nn.Identity()])
        self._qkv = None

    def _stacked(self):
        ps = [self.to_q.weight, self.to_k.weight, self.to_v.weight, self.to_q.bias, self.to_k.bias, self.to_v.bias]
        key = tuple((p._version, p.data_ptr()) for p in ps)
        if self._qkv is None or self._qkv[0] != key:
            self._qkv = (key, torch.cat([p.detach() for p in ps[:3]], 0).contiguous(), torch.cat([p.detach() for p in ps[3:]], 0).contiguous())
        return self._qkv[1], self._qkv[2]

    @torch.no_grad()
    def run(self, x_nhwc: torch.Tensor) -> torch.Tensor:
        _need_kernels(x_nhwc, self.to_q.weight, "MidBlockAttention")
        B, H, W, Cc = x_nhwc.shape
        gn = self.group_norm
        hn = lib.groupnorm_silu_nhwc(x_nhwc, gn.weight, gn.bias, torch.empty_like(x_nhwc), groups=gn.num_groups, eps=gn.eps, silu=False)
        w, b = self._stacked()
        qkv = lib.gemm(hn.view(B * H * W, Cc), w, b, torch.empty(B * H * W, 3 * Cc, dtype=torch.bfloat16, device=x_nhwc.device))
        q, k, v = qkv.view(B, 1, H * W, 3, Cc).unbind(3)                          # one head of dim C
        o = F.scaled_dot_product_attention(q, k, v)                                # PyTorch (see the section header)
        o = o.reshape(B * H * W, Cc).contiguous()
        out = lib.gemm(o, self.to_out[0].weight, self.to_out[0].bias, torch.empty_like(o))
        return out.view(B, H, W, Cc) + x_nhwc

    def forward(self, x: torch.Tensor, *args, **kwargs) -> torch.Tensor:
        return self.run(_nhwc(x)).permute(0, 3, 1, 2)


class _ResStack(nn.Module):
    """`resnets` (+ optional `upsamplers` / `downsamplers`) of one diffusers UpDecoderBlock2D / DownEncoderBlock2D."""

    def __init__(self, cin: int, cout: int, n: int, up: bool = False, down: bool = False, groups: int = 32):
        super().__init__()
        self.resnets = nn.ModuleList([DecoderResBlock(cin if i == 0 else cout, cout, groups) for i in range(n)])
        if up:
            self.upsamplers = nn.ModuleList([UpsampleConv(cout)])
        if down:
            self.downsamplers = nn.ModuleList([_Downsample(cout)])

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        for r in self.resnets:
            x = r(x)
        for m in getattr(self, "upsamplers", ()):
            x = m(x)
        for m in getattr(self, "downsamplers", ()):
            x = m(x)
        return x


class _Downsample(nn.Module):
    """diffusers `Downsample2D(padding=0)` of the VAE encoder: zero-pad right / bottom by one, 3x3 stride-2 convolution (PyTorch)."""

    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return F.conv2d(F.pad(x, (0, 1, 0, 1)), self.conv.weight, self.conv.bias, stride=2).contiguous(memory_format=torch.channels_last)


class _MidBlock(nn.Module):
    def __init__(self, channels: int, groups: int = 32):
        super().__init__()
        self.attentions = nn.ModuleList([MidBlockAttention(channels, groups)])
        self.resnets = nn.ModuleList([DecoderResBlock(channels, channels, groups), DecoderResBlock(channels, channels, groups)])

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.resnets[1](self.attentions[0](self.resnets[0](x)))


def _norm_act_conv(norm: nn.GroupNorm, conv: nn.Conv2d, x: torch.Tensor, cache: dict) -> torch.Tensor:
    """conv_norm_out -> SiLU -> conv_out tail shared by the encoder and the decoder (GroupNorm + SiLU on the kernel)."""
    xh = _nhwc(x)
    h = lib.groupnorm_silu_nhwc(xh, norm.weight, norm.bias, torch.empty_like(xh), groups=norm.num_groups, eps=norm.eps, silu=True)
    return _conv3x3(conv, h, cache).permute(0, 3, 1, 2)


class VaeDecoder(nn.Module):
    """diffusers `Decoder` of the SDXL-VAE: z (B, 4, h, w) -> image (B, 3, 8h, 8w)."""

    def __init__(self, cfg=SDXL_VAE_CONFIG):
        super().__init__()
        ch, n, g = list(cfg["block_out_channels"]), cfg["layers_per_block"], cfg["norm_num_groups"]
        rev = ch[::-1]
        self.conv_in = nn.Conv2d(cfg["latent_channels"], rev[0], 3, padding=1)
        self.mid_block = _MidBlock(rev[0], g)
        self.up_blocks = nn.ModuleList([_ResStack(rev[max(i - 1, 0)], rev[i], n + 1, up=i < len(rev) - 1, groups=g)
                                        for i in range(len(rev))])
        self.conv_norm_out = nn.GroupNorm(g, ch[0], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[0], cfg["out_channels"], 3, padding=1)
        self._cache = {}

    def _trunk(self, z: torch.Tensor) -> torch.Tensor:
        """conv_in -> mid block -> up blocks: everything before conv_norm_out."""
        _need_kernels(z, self.conv_in.weight, "VaeDecoder")
        x = F.conv2d(z.to(torch.bfloat16), self.conv_in.weight, self.conv_in.bias, padding=1).contiguous(memory_format=torch.channels_last)
        x = self.mid_block(x)
        for blk in self.up_blocks:
            x = blk(x)
        return x

    @torch.no_grad()
    def forward(self, z: torch.Tensor) -> torch.Tensor:
        return _norm_act_conv(self.conv_norm_out, self.conv_out, self._trunk(z), self._cache)

    @torch.no_grad()
    def forward_uint8(self, z: torch.Tensor, return_float: bool = False):
        """z (B, 4, h, w) -> (uint8 pixels (B, H, W, 3), conv_out's fp32 output (B, H, W, 3) or None): conv_norm_out + SiLU on
        the GroupNorm kernel, then conv_out and save_image's conversion in one `pxa_vae_out_u8` pass."""
        xh = _nhwc(self._trunk(z))
        norm, conv = self.conv_norm_out, self.conv_out
        h = lib.groupnorm_silu_nhwc(xh, norm.weight, norm.bias, torch.empty_like(xh), groups=norm.num_groups, eps=norm.eps, silu=True)
        key = (conv.weight._version, conv.weight.data_ptr(), conv.bias._version, conv.bias.data_ptr())
        if self._cache.get("u8_key") != key:
            self._cache["u8_key"] = key
            self._cache["u8_w"] = conv.weight.detach().to(torch.bfloat16).permute(0, 2, 3, 1).contiguous()
            self._cache["u8_b"] = conv.bias.detach().float().contiguous()
        B, H, W, _ = h.shape
        out = torch.empty(B, H, W, 3, dtype=torch.uint8, device=h.device)
        y = torch.empty(B, H, W, 3, dtype=torch.float32, device=h.device) if return_float else None
        return lib.vae_out_u8(h, self._cache["u8_w"], self._cache["u8_b"], out, y), y


class VaeEncoder(nn.Module):
    """diffusers `Encoder` of the SDXL-VAE: image (B, 3, H, W) -> moments (B, 8, H/8, W/8) (train.py:149 `vae.encode`)."""

    def __init__(self, cfg=SDXL_VAE_CONFIG):
        super().__init__()
        ch, n, g = list(cfg["block_out_channels"]), cfg["layers_per_block"], cfg["norm_num_groups"]
        self.conv_in = nn.Conv2d(cfg["in_channels"], ch[0], 3, padding=1)
        self.down_blocks = nn.ModuleList([_ResStack(ch[max(i - 1, 0)], ch[i], n, down=i < len(ch) - 1, groups=g) for i in range(len(ch))])
        self.mid_block = _MidBlock(ch[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[-1], 2 * cfg["latent_channels"], 3, padding=1)
        self._cache = {}

    @torch.no_grad()
    def forward(self, img: torch.Tensor) -> torch.Tensor:
        _need_kernels(img, self.conv_in.weight, "VaeEncoder")
        x = F.conv2d(img.to(torch.bfloat16), self.conv_in.weight, self.conv_in.bias, padding=1).contiguous(memory_format=torch.channels_last)
        for blk in self.down_blocks:
            x = blk(x)
        x = self.mid_block(x)
        return _norm_act_conv(self.conv_norm_out, self.conv_out, x, self._cache)


class _Sample:
    def __init__(self, sample):
        self.sample = sample


class DiagonalGaussian:
    """diffusers `DiagonalGaussianDistribution` (`vae.encode(x).latent_dist`, train.py:149)."""

    def __init__(self, moments: torch.Tensor):
        self.mean, logvar = moments.float().chunk(2, dim=1)
        self.logvar = logvar.clamp(-30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self, generator=None) -> torch.Tensor:
        dev = self.mean.device                              # a CPU generator with CUDA moments: draw where the generator lives (diffusers' randn_tensor)
        gdev = generator.device if generator is not None else dev
        noise = torch.randn(self.mean.shape, generator=generator, device=gdev, dtype=self.mean.dtype).to(dev)
        return self.mean + self.std * noise

    def mode(self) -> torch.Tensor:
        return self.mean


class _Latent:
    def __init__(self, dist):
        self.latent_dist = dist


class AutoencoderKL(nn.Module):
    """Drop-in for the two calls the reference makes on diffusers' AutoencoderKL: `vae.decode(z / scaling_factor).sample`
    (scripts/inference.py:136) and `vae.encode(img).latent_dist.sample()` (train_scripts/train.py:149), with the same state-dict
    keys and `config.scaling_factor`."""

    def __init__(self, cfg=SDXL_VAE_CONFIG):
        super().__init__()
        self.encoder, self.decoder = VaeEncoder(cfg), VaeDecoder(cfg)
        lc = cfg["latent_channels"]
        self.quant_conv = nn.Conv2d(2 * lc, 2 * lc, 1)
        self.post_quant_conv = nn.Conv2d(lc, lc, 1)
        self.config = type("Config", (), dict(cfg))()

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True):
        z = F.conv2d(z.to(self.post_quant_conv.weight.dtype), self.post_quant_conv.weight, self.post_quant_conv.bias)
        img = self.decoder(z)
        return _Sample(img) if return_dict else (img,)

    @torch.no_grad()
    def decode_to_uint8(self, z: torch.Tensor, return_float: bool = False):
        """`decode(z).sample` written straight to image bytes: uint8 (B, H, W, 3) on the device, equal to what
        torchvision's `save_image(img, normalize=True, value_range=(-1, 1))` makes of the decoded image (before the JPEG
        encoder).  The decoder's conv_out and the conversion run as one kernel (`pxa_vae_out_u8`).  With return_float, also
        returns conv_out's fp32 output as a (B, 3, H, W) view of an NHWC tensor."""
        z = F.conv2d(z.to(self.post_quant_conv.weight.dtype), self.post_quant_conv.weight, self.post_quant_conv.bias)
        if self.decoder.conv_out.out_channels != 3:
            raise ValueError("decode_to_uint8 needs a decoder with 3 output channels")
        u8, y = self.decoder.forward_uint8(z, return_float)
        return (u8, y.permute(0, 3, 1, 2)) if return_float else u8

    @torch.no_grad()
    def encode(self, img: torch.Tensor, return_dict: bool = True):
        m = self.encoder(img)
        m = F.conv2d(m.to(self.quant_conv.weight.dtype), self.quant_conv.weight, self.quant_conv.bias)
        dist = DiagonalGaussian(m)
        return _Latent(dist) if return_dict else (dist,)
