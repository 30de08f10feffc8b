"""ORACLE (test infrastructure, not product code): plain-PyTorch restatement of the reference causal-VAE DECODE path.

Restates `CausalVideoVAE.decode` (video_vae/modeling_causal_vae.py:376-395) for the un-tiled case as pure functions over
a state-dict in the reference key layout:
  V = video_vae/modeling_causal_vae.py     D = .../modeling_enc_dec.py     K = .../modeling_block.py
  R = .../modeling_resnet.py               C = .../modeling_causal_conv.py
plus the mid-block attention from diffusers 0.30 `Attention(_from_deprecated_attn_block=True)` (not in the reference checkout;
pinned version diffusers>=0.30.1, requirements.txt:6; call sites K:413-427, K:458).

Temporal chunking with the 2-frame feature cache (C:126-143, V:346-374) is EXACT w.r.t. the un-chunked computation
(causal convs + per-frame GroupNorm), so this restatement computes the whole clip at once; tests/golden pins it against the
reference's `decode(temporal_chunk=False)` AND `chunk_decode(window_size=1|2)`.
Spatial tiling (V:468-519) is restated separately in `tiled_decode` (tiles are decoded independently and cross-faded).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Tuple

import torch
import torch.nn.functional as F

Params = Dict[str, torch.Tensor]


@dataclass
class VaeDecoderConfig:
    """Decoder-side constructor arguments of CausalVideoVAE (V:73-116)."""
    latent_channels: int = 16
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: Tuple[int, ...] = (3, 3, 3, 3)
    spatial_up_sample: Tuple[bool, ...] = (True, True, True, False)
    temporal_up_sample: Tuple[bool, ...] = (True, True, True, False)
    norm_num_groups: int = 32


def causal_conv3d(p: Params, pre: str, x: torch.Tensor, stride=(1, 1, 1)) -> torch.Tensor:
    """CausalConv3d.forward, non-chunked (C:116-125,145): zero pad (k-1) frames in front, k//2 each side spatially;
    `stride` = (t, h, w) of the down-samplers (C:66-67, R:322, R:486)."""
    w, b = p[pre + ".conv.weight"], p.get(pre + ".conv.bias")
    kt, kh, kw = w.shape[2:]
    x = F.pad(x, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0))
    return F.conv3d(x, w, b, stride=stride)


def causal_group_norm(p: Params, pre: str, x: torch.Tensor, groups: int) -> torch.Tensor:
    """CausalGroupNorm (C:36-43): GroupNorm applied to every frame separately, eps 1e-6, affine."""
    b, c, t, h, w = x.shape
    y = F.group_norm(x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w), groups, p[pre + ".weight"], p[pre + ".bias"], 1e-6)
    return y.reshape(b, t, c, h, w).permute(0, 2, 1, 3, 4)


def resnet_block(p: Params, pre: str, x: torch.Tensor, groups: int) -> torch.Tensor:
    """CausalResnetBlock3D.forward (R:115-150), output_scale_factor = 1, no temb."""
    h = causal_conv3d(p, pre + ".conv1", F.silu(causal_group_norm(p, pre + ".norm1", x, groups)))
    h = causal_conv3d(p, pre + ".conv2", F.silu(causal_group_norm(p, pre + ".norm2", h, groups)))
    if (pre + ".conv_shortcut.conv.weight") in p:
        x = causal_conv3d(p, pre + ".conv_shortcut", x)
    return x + h


def mid_attention(p: Params, pre: str, x: torch.Tensor, groups: int) -> torch.Tensor:
    """Per-frame single-head spatial attention (K:454-460 + diffusers Attention, deprecated-attn-block form)."""
    b, c, t, h, w = x.shape
    f = x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h * w)                 # (b t) c (h w)
    res = f
    n = F.group_norm(f, groups, p[pre + ".group_norm.weight"], p[pre + ".group_norm.bias"], 1e-6).transpose(1, 2)
    q = F.linear(n, p[pre + ".to_q.weight"], p[pre + ".to_q.bias"])
    k = F.linear(n, p[pre + ".to_k.weight"], p[pre + ".to_k.bias"])
    v = F.linear(n, p[pre + ".to_v.weight"], p[pre + ".to_v.bias"])
    o = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None])[:, 0]
    o = F.linear(o, p[pre + ".to_out.0.weight"], p[pre + ".to_out.0.bias"]).transpose(1, 2)
    return (o + res).reshape(b, t, c, h, w).permute(0, 2, 1, 3, 4)


def spatial_upsample(p: Params, pre: str, x: torch.Tensor) -> torch.Tensor:
    """CausalUpsample2x (R:609-617): conv C->4C then 'b (c p1 p2) t h w -> b c t (h p1) (w p2)'."""
    y = causal_conv3d(p, pre + ".conv", x)
    b, c4, t, h, w = y.shape
    c = c4 // 4
    y = y.reshape(b, c, 2, 2, t, h, w).permute(0, 1, 4, 5, 2, 6, 3)
    return y.reshape(b, c, t, h * 2, w * 2)


def temporal_upsample(p: Params, pre: str, x: torch.Tensor, is_init_image: bool = True) -> torch.Tensor:
    """CausalTemporalUpsample2x (R:716-729): conv C->2C, 'b (c p) t h w -> b c (t p) h w', drop the first frame of a clip
    that starts with the image frame."""
    y = causal_conv3d(p, pre + ".conv", x)
    b, c2, t, h, w = y.shape
    c = c2 // 2
    y = y.reshape(b, c, 2, t, h, w).permute(0, 1, 3, 2, 4, 5).reshape(b, c, 2 * t, h, w)
    return y[:, :, 1:] if is_init_image else y


def decoder_forward(p: Params, cfg: VaeDecoderConfig, z: torch.Tensor) -> torch.Tensor:
    """CausalVaeDecoder.forward (D:302-366), whole clip at once (is_init_image=True)."""
    g = cfg.norm_num_groups
    x = causal_conv3d(p, "decoder.conv_in", z)
    x = resnet_block(p, "decoder.mid_block.resnets.0", x, g)
    x = mid_attention(p, "decoder.mid_block.attentions.0", x, g)
    x = resnet_block(p, "decoder.mid_block.resnets.1", x, g)
    n_blocks = len(cfg.block_out_channels)
    for i in range(n_blocks):
        for j in range(cfg.layers_per_block[i]):
            x = resnet_block(p, f"decoder.up_blocks.{i}.resnets.{j}", x, g)
        if cfg.spatial_up_sample[i]:
            x = spatial_upsample(p, f"decoder.up_blocks.{i}.upsamplers.0", x)
        if cfg.temporal_up_sample[i]:
            x = temporal_upsample(p, f"decoder.up_blocks.{i}.temporal_upsamplers.0", x, True)
    x = F.silu(causal_group_norm(p, "decoder.conv_norm_out", x, g))
    return causal_conv3d(p, "decoder.conv_out", x)


def decode(p: Params, cfg: VaeDecoderConfig, z: torch.Tensor) -> torch.Tensor:
    """CausalVideoVAE.decode, un-tiled (V:386-390): post_quant_conv (1x1x1) then the decoder."""
    return decoder_forward(p, cfg, causal_conv3d(p, "post_quant_conv", z))


def _blend_v(a, b, extent):
    extent = min(a.shape[3], b.shape[3], extent)
    for y in range(extent):
        b[:, :, :, y, :] = a[:, :, :, -extent + y, :] * (1 - y / extent) + b[:, :, :, y, :] * (y / extent)
    return b


def _blend_h(a, b, extent):
    extent = min(a.shape[4], b.shape[4], extent)
    for x in range(extent):
        b[:, :, :, :, x] = a[:, :, :, :, -extent + x] * (1 - x / extent) + b[:, :, :, :, x] * (x / extent)
    return b


def tiled_decode(p: Params, cfg: VaeDecoderConfig, z: torch.Tensor, tile_sample_min_size: int = 256,
                 overlap_factor: float = 0.25, downsample: int = 8) -> torch.Tensor:
    """CausalVideoVAE.tiled_decode (V:468-519) with blend_v/blend_h (V:397-407)."""
    tile_latent = int(tile_sample_min_size / downsample)
    overlap = int(tile_latent * (1 - overlap_factor))
    extent = int(tile_sample_min_size * overlap_factor)
    limit = tile_sample_min_size - extent
    rows = []
    for i in range(0, z.shape[3], overlap):
        row = []
        for j in range(0, z.shape[4], overlap):
            row.append(decode(p, cfg, z[:, :, :, i:i + tile_latent, j:j + tile_latent]))
        rows.append(row)
    out_rows = []
    for i, row in enumerate(rows):
        res = []
        for j, tile in enumerate(row):
            if i > 0:
                tile = _blend_v(rows[i - 1][j], tile, extent)
            if j > 0:
                tile = _blend_h(row[j - 1], tile, extent)
            res.append(tile[:, :, :, :limit, :limit])
        out_rows.append(torch.cat(res, dim=4))
    return torch.cat(out_rows, dim=3)


# ---- encoder (i2v image latent: pipeline P:911) ------------------------------------------------------------------------
@dataclass
class VaeEncoderConfig:
    """Encoder-side constructor arguments of CausalVideoVAE (V:76-93)."""
    in_channels: int = 3
    latent_channels: int = 16
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: Tuple[int, ...] = (2, 2, 2, 2)
    spatial_down_sample: Tuple[bool, ...] = (True, True, True, False)
    temporal_down_sample: Tuple[bool, ...] = (True, True, True, False)
    norm_num_groups: int = 32


def encoder_forward(p: Params, cfg: VaeEncoderConfig, x: torch.Tensor) -> torch.Tensor:
    """CausalVaeEncoder.forward (D:149-198), whole clip at once (is_init_image=True): conv_in, down blocks (resnets, then the
    stride-(1,2,2) and stride-(2,1,1) causal convs K:528-540), mid block, GroupNorm+SiLU, conv_out (2*latent channels)."""
    g = cfg.norm_num_groups
    h = causal_conv3d(p, "encoder.conv_in", x)
    for i in range(len(cfg.block_out_channels)):
        for j in range(cfg.layers_per_block[i]):
            h = resnet_block(p, f"encoder.down_blocks.{i}.resnets.{j}", h, g)
        if cfg.spatial_down_sample[i]:
            h = causal_conv3d(p, f"encoder.down_blocks.{i}.downsamplers.0.conv", h, stride=(1, 2, 2))
        if cfg.temporal_down_sample[i]:
            h = causal_conv3d(p, f"encoder.down_blocks.{i}.temporal_downsamplers.0.conv", h, stride=(2, 1, 1))
    h = resnet_block(p, "encoder.mid_block.resnets.0", h, g)
    h = mid_attention(p, "encoder.mid_block.attentions.0", h, g)
    h = resnet_block(p, "encoder.mid_block.resnets.1", h, g)
    h = F.silu(causal_group_norm(p, "encoder.conv_norm_out", h, g))
    return causal_conv3d(p, "encoder.conv_out", h)


def encode_moments(p: Params, cfg: VaeEncoderConfig, x: torch.Tensor) -> torch.Tensor:
    """CausalVideoVAE.encode, un-tiled, un-chunked (V:300-303): encoder then quant_conv (1x1x1); returns the moments
    [B, 2*latent, T', h, w]: mean = first half, logvar = second half clamped to [-30, 20] (D:372-373)."""
    return causal_conv3d(p, "quant_conv", encoder_forward(p, cfg, x))


def vae_encoder_param_shapes(cfg: VaeEncoderConfig) -> Dict[str, tuple]:
    s: Dict[str, tuple] = {}

    def conv(name, co, ci, k):
        s[name + ".conv.weight"] = (co, ci, k, k, k)
        s[name + ".conv.bias"] = (co,)

    def norm(name, c):
        s[name + ".weight"] = (c,)
        s[name + ".bias"] = (c,)

    def res(name, ci, co):
        norm(name + ".norm1", ci); conv(name + ".conv1", co, ci, 3)
        norm(name + ".norm2", co); conv(name + ".conv2", co, co, 3)
        if ci != co:
            conv(name + ".conv_shortcut", co, ci, 1)

    conv("encoder.conv_in", cfg.block_out_channels[0], cfg.in_channels, 3)
    prev = cfg.block_out_channels[0]
    for i, co in enumerate(cfg.block_out_channels):
        for j in range(cfg.layers_per_block[i]):
            res(f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else co, co)
        if cfg.spatial_down_sample[i]:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", co, co, 3)
        if cfg.temporal_down_sample[i]:
            conv(f"encoder.down_blocks.{i}.temporal_downsamplers.0.conv", co, co, 3)
        prev = co
    top = cfg.block_out_channels[-1]
    res("encoder.mid_block.resnets.0", top, top)
    norm("encoder.mid_block.attentions.0.group_norm", top)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        s[f"encoder.mid_block.attentions.0.{n}.weight"] = (top, top)
        s[f"encoder.mid_block.attentions.0.{n}.bias"] = (top,)
    res("encoder.mid_block.resnets.1", top, top)
    norm("encoder.conv_norm_out", top)
    conv("encoder.conv_out", 2 * cfg.latent_channels, top, 3)
    conv("quant_conv", 2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)
    return s


# ------------------------------------------------------------------------------------------------------------------
def vae_decoder_param_shapes(cfg: VaeDecoderConfig) -> Dict[str, tuple]:
    s: Dict[str, tuple] = {}

    def conv(name, co, ci, k):
        s[name + ".conv.weight"] = (co, ci, k, k, k)
        s[name + ".conv.bias"] = (co,)

    def norm(name, c):
        s[name + ".weight"] = (c,)
        s[name + ".bias"] = (c,)

    def res(name, ci, co):
        norm(name + ".norm1", ci); conv(name + ".conv1", co, ci, 3)
        norm(name + ".norm2", co); conv(name + ".conv2", co, co, 3)
        if ci != co:
            conv(name + ".conv_shortcut", co, ci, 1)

    rev = list(reversed(cfg.block_out_channels))
    top = rev[0]
    conv("post_quant_conv", cfg.latent_channels, cfg.latent_channels, 1)
    conv("decoder.conv_in", top, cfg.latent_channels, 3)
    res("decoder.mid_block.resnets.0", top, top)
    norm("decoder.mid_block.attentions.0.group_norm", top)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        s[f"decoder.mid_block.attentions.0.{n}.weight"] = (top, top)
        s[f"decoder.mid_block.attentions.0.{n}.bias"] = (top,)
    res("decoder.mid_block.resnets.1", top, top)
    prev = top
    for i, co in enumerate(rev):
        for j in range(cfg.layers_per_block[i]):
            res(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else co, co)
        if cfg.spatial_up_sample[i]:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", 4 * co, co, 3)
        if cfg.temporal_up_sample[i]:
            conv(f"decoder.up_blocks.{i}.temporal_upsamplers.0.conv", 2 * co, co, 3)
        prev = co
    norm("decoder.conv_norm_out", cfg.block_out_channels[0])
    conv("decoder.conv_out", cfg.out_channels, cfg.block_out_channels[0], 3)
    return s


def synthetic_vae_params(cfg, seed: int = 0, device: str = "cpu", bf16_representable: bool = True) -> Params:
    """Seeded parameters: conv/linear weights N(0, 1/fan_in) (x0.5 on each residual branch's last conv so activations stay
    O(1) through ~30 residual blocks), biases N(0, 0.02^2), GroupNorm weight 1+N(0,0.1^2), bias N(0,0.05^2).
    `cfg`: VaeDecoderConfig (decoder + post_quant_conv keys) or VaeEncoderConfig (encoder + quant_conv keys)."""
    g = torch.Generator().manual_seed(seed)
    out: Params = {}
    shapes = vae_encoder_param_shapes(cfg) if isinstance(cfg, VaeEncoderConfig) else vae_decoder_param_shapes(cfg)
    for name, shp in shapes.items():
        if len(shp) >= 2:
            fan_in = 1
            for d in shp[1:]:
                fan_in *= d
            std = fan_in ** -0.5
            if ".conv2." in name or "to_out" in name:
                std *= 0.5
            w = torch.randn(shp, generator=g) * std
            if bf16_representable:
                w = w.bfloat16().float()
            out[name] = w.to(device)
        elif ("norm" in name) and name.endswith("weight"):
            out[name] = (1.0 + 0.1 * torch.randn(shp, generator=g)).to(device)
        elif "norm" in name:
            out[name] = (0.05 * torch.randn(shp, generator=g)).to(device)
        else:
            out[name] = (0.02 * torch.randn(shp, generator=g)).to(device)
    return out
