"""ORACLE (test infrastructure, not product code): plain-PyTorch restatement of the reference causal-VAE ENCODE paths for
video clips, on top of the un-chunked restatement in `oracle.vae_oracle`:
  * `chunk_encode_moments`: CausalVideoVAE.chunk_encode (video_vae/modeling_causal_vae.py:311-341) with the per-conv
    feature cache of CausalConv3d (video_vae/modeling_causal_conv.py:126-145), including the stride-2 temporal
    down-sampler's one-frame context (C:140-141);
  * `tiled_encode_moments`: CausalVideoVAE.tiled_encode (V:409-466) with blend_v / blend_h (V:397-407).
Pinned to the unmodified reference by tests/golden/vae_encoder_video_small.pt (oracle/pin/make_encode_golden.py).

Only tests/ may import this module.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle.vae_oracle import (Params, VaeEncoderConfig, _blend_h, _blend_v, causal_group_norm, encode_moments,
                               mid_attention)


def _cached_conv3d(p: Params, pre: str, x: torch.Tensor, cache: Dict[str, torch.Tensor], first: bool,
                   stride=(1, 1, 1)) -> torch.Tensor:
    """CausalConv3d.forward with temporal_chunk=True (C:126-145): the first chunk is zero-padded in front; a later chunk of
    a kt=3 conv gets the 2 cached frames prepended (stride 1) or only the last one (stride-2 temporal down-sampler,
    C:140-141).  The cache becomes the last 2 frames of the (padded / prepended) input."""
    w, b = p[pre + ".conv.weight"], p.get(pre + ".conv.bias")
    kt, kh, kw = w.shape[2:]
    x = F.pad(x, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1 if first else 0, 0))
    if not first and kt == 3:
        ctx = cache[pre]
        x = torch.cat([ctx if stride[0] == 1 else ctx[:, :, -1:], x], dim=2)
    cache[pre] = x[:, :, -2:].clone()
    return F.conv3d(x, w, b, stride=stride)


def _cached_resnet_block(p: Params, pre: str, x: torch.Tensor, groups: int, cache, first: bool) -> torch.Tensor:
    h = _cached_conv3d(p, pre + ".conv1", F.silu(causal_group_norm(p, pre + ".norm1", x, groups)), cache, first)
    h = _cached_conv3d(p, pre + ".conv2", F.silu(causal_group_norm(p, pre + ".norm2", h, groups)), cache, first)
    if (pre + ".conv_shortcut.conv.weight") in p:
        x = _cached_conv3d(p, pre + ".conv_shortcut", x, cache, first)
    return x + h


def chunk_encode_moments(p: Params, cfg: VaeEncoderConfig, x: torch.Tensor, window_size: int = 16) -> torch.Tensor:
    """CausalVideoVAE.chunk_encode (V:311-341): chunks [0, window+1), then `window` frames each (the last takes the rest),
    each through the encoder and quant_conv with the per-conv feature cache; moments concatenated over time."""
    g, n = cfg.norm_num_groups, x.shape[2]
    bounds = [(0, min(n, window_size + 1))]
    while bounds[-1][1] < n:
        bounds.append((bounds[-1][1], min(n, bounds[-1][1] + window_size)))
    cache: Dict[str, torch.Tensor] = {}
    outs = []
    for ci, (a, b) in enumerate(bounds):
        first = ci == 0
        h = _cached_conv3d(p, "encoder.conv_in", x[:, :, a:b], cache, first)
        for i in range(len(cfg.block_out_channels)):
            for j in range(cfg.layers_per_block[i]):
                h = _cached_resnet_block(p, f"encoder.down_blocks.{i}.resnets.{j}", h, g, cache, first)
            if cfg.spatial_down_sample[i]:
                h = _cached_conv3d(p, f"encoder.down_blocks.{i}.downsamplers.0.conv", h, cache, first, stride=(1, 2, 2))
            if cfg.temporal_down_sample[i]:
                h = _cached_conv3d(p, f"encoder.down_blocks.{i}.temporal_downsamplers.0.conv", h, cache, first,
                                   stride=(2, 1, 1))
        h = _cached_resnet_block(p, "encoder.mid_block.resnets.0", h, g, cache, first)
        h = mid_attention(p, "encoder.mid_block.attentions.0", h, g)
        h = _cached_resnet_block(p, "encoder.mid_block.resnets.1", h, g, cache, first)
        h = _cached_conv3d(p, "encoder.conv_out", F.silu(causal_group_norm(p, "encoder.conv_norm_out", h, g)), cache, first)
        outs.append(_cached_conv3d(p, "quant_conv", h, cache, first))
    return torch.cat(outs, dim=2)


def tiled_encode_moments(p: Params, cfg: VaeEncoderConfig, x: torch.Tensor, tile_sample_min_size: int = 256,
                         window_size=None, overlap_factor: float = 0.25, downsample: int = 8) -> torch.Tensor:
    """CausalVideoVAE.tiled_encode (V:409-466) with blend_v/blend_h (V:397-407); each pixel tile is chunk-encoded when
    `window_size` is given (temporal_chunk=True), else encoded whole."""
    tile_latent = int(tile_sample_min_size / downsample)
    overlap = int(tile_sample_min_size * (1 - overlap_factor))
    extent = int(tile_latent * overlap_factor)
    limit = tile_latent - extent
    rows = []
    for i in range(0, x.shape[3], overlap):
        row = []
        for j in range(0, x.shape[4], overlap):
            tile = x[:, :, :, i:i + tile_sample_min_size, j:j + tile_sample_min_size]
            row.append(encode_moments(p, cfg, tile) if window_size is None else chunk_encode_moments(p, cfg, tile, window_size))
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
