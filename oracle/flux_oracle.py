"""ORACLE (test infrastructure, not product code): plain-PyTorch restatement of the reference miniFLUX DiT step.

Restates `PyramidFluxTransformer.forward` (pyramid_dit/flux_modules/modeling_pyramid_flux.py:392-542) for the default
inference path (no sequence parallel, use_flash_attn=False, use_temporal_causal=True, one stage per call) as pure
functions over a state-dict in the reference's key layout.  Every function cites the reference lines it follows:
  F = pyramid_dit/flux_modules/modeling_pyramid_flux.py      B = .../modeling_flux_block.py
  N = .../modeling_normalization.py                          E = .../modeling_embedding.py

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
Parity status: PINNED against the unmodified reference imported through oracle/pin/ref_shim.py
(oracle/pin/make_golden.py -> tests/golden/flux_*.pt, checked by tests/test_oracle_golden.py).

The same code serves two numerics modes:
  * fp32 (default): the "truth" the CUDA path is compared with;
  * under `torch.autocast(device, torch.bfloat16)`: reproduces the reference's own bf16 dtype policy because
    it uses the same torch ops the reference uses (F.linear, F.layer_norm, F.scaled_dot_product_attention, ...).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

Params = Dict[str, torch.Tensor]
HEAD_CHUNK = 0   # >0: run SDPA over this many heads at a time (bounds the S x S score memory at full size)


@dataclass
class FluxConfig:
    """Constructor arguments of PyramidFluxTransformer that shape the computation (F:80-96)."""
    num_layers: int = 8
    num_single_layers: int = 16
    num_attention_heads: int = 30
    attention_head_dim: int = 64
    in_channels: int = 64
    joint_attention_dim: int = 4096
    pooled_projection_dim: int = 768
    axes_dims_rope: Sequence[int] = (16, 24, 24)
    patch_size: int = 2  # hard-coded F:147

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim


# ------------------------------------------------------------------------------------------------------------------
# conditioning
# ------------------------------------------------------------------------------------------------------------------
def timestep_embedding(t: torch.Tensor, dim: int = 256) -> torch.Tensor:
    """get_timestep_embedding with flip_sin_to_cos=True, downscale_freq_shift=0, scale=1 (E:11-62, E:188)."""
    half = dim // 2
    exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32, device=t.device) / half
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


def linear(p: Params, prefix: str, x: torch.Tensor) -> torch.Tensor:
    return F.linear(x, p[prefix + ".weight"], p.get(prefix + ".bias"))


def time_text_embed(p: Params, timestep: torch.Tensor, pooled: torch.Tensor) -> torch.Tensor:
    """CombinedTimestepTextProjEmbeddings.forward (E:193-201): TimestepEmbedding (E:112-129) + PixArtAlphaTextProjection
    with SiLU (E:154-158)."""
    proj = timestep_embedding(timestep, 256).to(pooled.dtype)  # E:195
    h = linear(p, "time_text_embed.timestep_embedder.linear_1", proj)
    h = linear(p, "time_text_embed.timestep_embedder.linear_2", F.silu(h))
    c = linear(p, "time_text_embed.text_embedder.linear_1", pooled)
    c = linear(p, "time_text_embed.text_embedder.linear_2", F.silu(c))
    return h + c


# ------------------------------------------------------------------------------------------------------------------
# ids, RoPE, mask (merge_input, F:239-352)
# ------------------------------------------------------------------------------------------------------------------
def clip_ids(temp: int, height: int, width: int, train_height: int, train_width: int, start_time: int) -> torch.Tensor:
    """_prepare_image_ids (F:186-211) for one clip, without the batch dimension: [(t h w), 3] float32."""
    ids = torch.zeros(temp, height, width, 3)
    ids[..., 0] += torch.arange(start_time, start_time + temp)[:, None, None]
    if height != train_height:
        hp = F.interpolate(torch.arange(train_height)[None, None, :].float(), height, mode="linear").squeeze(0).squeeze(0)
    else:
        hp = torch.arange(train_height).float()
    ids[..., 1] += hp[None, :, None]
    if width != train_width:
        wp = F.interpolate(torch.arange(train_width)[None, None, :].float(), width, mode="linear").squeeze(0).squeeze(0)
    else:
        wp = torch.arange(train_width).float()
    ids[..., 2] += wp[None, None, :]
    return ids.reshape(-1, 3)


def sequence_ids(clip_shapes: Sequence[Sequence[int]], text_len: int, patch: int = 2) -> torch.Tensor:
    """[text ; clip_0 ; ... ; clip_n] position ids [S, 3] (F:214-237, F:266-269): text ids are (0,0,0); the time id runs
    over clips; coarser clips get spatial positions interpolated onto the finest (= last) clip's grid."""
    th, tw = clip_shapes[-1][-2] // patch, clip_shapes[-1][-1] // patch
    out = [torch.zeros(text_len, 3)]
    start = 0
    for shp in clip_shapes:
        t, h, w = shp[-3], shp[-2] // patch, shp[-1] // patch
        out.append(clip_ids(t, h, w, th, tw, start))
        start += t
    return torch.cat(out, 0)


def rope_table(ids: torch.Tensor, axes_dim: Sequence[int], theta: float = 10000.0) -> torch.Tensor:
    """EmbedND / rope (F:28-57): float64 angles, returns (cos, sin) [S, sum(axes)/2, 2] float32.
    The reference materialises [[cos, -sin], [sin, cos]]; (cos, sin) carries the same information."""
    outs = []
    for i, d in enumerate(axes_dim):
        scale = torch.arange(0, d, 2, dtype=torch.float64) / d
        omega = 1.0 / (theta ** scale)
        ang = ids[:, i].double()[:, None] * omega[None, :]
        outs.append(torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1))
    return torch.cat(outs, dim=1).float()


def apply_rope(x: torch.Tensor, cs: torch.Tensor) -> torch.Tensor:
    """apply_rope (B:34-39) on x [B, S, H, hd] with cs [S, hd/2, 2]: interleaved pairs, fp32, cast back (`type_as`)."""
    x_ = x.float().reshape(*x.shape[:-1], -1, 2)
    c = cs[None, :, None, :, 0].to(x.device)
    s = cs[None, :, None, :, 1].to(x.device)
    o0 = c * x_[..., 0] - s * x_[..., 1]
    o1 = s * x_[..., 0] + c * x_[..., 1]
    return torch.stack([o0, o1], dim=-1).reshape(*x.shape).type_as(x)


def token_segments(encoder_attention_mask: torch.Tensor, video_len: int) -> torch.Tensor:
    """Segment id per token [B, S] (F:318-330): sample index + 1 for video and valid text tokens, 0 for padded text."""
    b, t = encoder_attention_mask.shape
    ids = torch.arange(1, b + 1, dtype=torch.int64)[:, None].repeat(1, t + video_len)
    ids[:, :t][encoder_attention_mask.cpu() == 0] = 0
    return ids


def attention_mask(seg: torch.Tensor, time_ids: torch.Tensor) -> torch.Tensor:
    """Dense bool mask [B, 1, S, S] = (same segment) & (time_q >= time_kv) (F:341-349)."""
    same = seg[:, :, None] == seg[:, None, :]
    causal = time_ids[:, None] >= time_ids[None, :]
    return (same & causal[None])[:, None]


# ------------------------------------------------------------------------------------------------------------------
# blocks
# ------------------------------------------------------------------------------------------------------------------
def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """RMSNorm.forward (N:66-79): fp32 variance; cast to the weight's dtype only if that is half precision."""
    var = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
    x = x * torch.rsqrt(var + eps)
    if weight.dtype in (torch.float16, torch.bfloat16):
        x = x.to(weight.dtype)
    return x * weight


def layer_norm(x: torch.Tensor) -> torch.Tensor:
    return F.layer_norm(x, (x.shape[-1],), None, None, 1e-6)


def joint_attention(q, k, v, cs, mask, heads):
    """VarlenSelfAttentionWithT5Mask / VarlenSelfAttnSingle for one stage (B:328-376, B:568-606):
    q,k,v [B, S, H, hd] -> rope(q,k) -> SDPA(mask) -> [B, S, H*hd]."""
    q = apply_rope(q, cs)
    k = apply_rope(k, cs)
    hc = HEAD_CHUNK or q.shape[2]          # memory knob for full-size runs (identical arithmetic per head)
    outs = []
    for h0 in range(0, q.shape[2], hc):
        sl = slice(h0, h0 + hc)
        outs.append(F.scaled_dot_product_attention(q[:, :, sl].transpose(1, 2), k[:, :, sl].transpose(1, 2),
                                                   v[:, :, sl].transpose(1, 2), dropout_p=0.0, is_causal=False,
                                                   attn_mask=mask).transpose(1, 2))
    return torch.cat(outs, dim=2).flatten(2, 3)


def double_block(p: Params, pre: str, x, ctx, temb, cs, mask, heads):
    """FluxTransformerBlock.forward (B:992-1044) + AdaLayerNormZero (N:150-193) + FluxAttnProcessor2_0 (B:805-874)."""
    b, lv, d = x.shape
    hd = d // heads
    sh_a, sc_a, g_a, sh_m, sc_m, g_m = linear(p, pre + ".norm1.linear", F.silu(temb)).chunk(6, dim=1)
    csh_a, csc_a, cg_a, csh_m, csc_m, cg_m = linear(p, pre + ".norm1_context.linear", F.silu(temb)).chunk(6, dim=1)
    xn = layer_norm(x) * (1 + sc_a[:, None]) + sh_a[:, None]
    cn = layer_norm(ctx) * (1 + csc_a[:, None]) + csh_a[:, None]

    def heads_view(t):
        return t.view(b, -1, heads, hd)

    q = rms_norm(heads_view(linear(p, pre + ".attn.to_q", xn)), p[pre + ".attn.norm_q.weight"])
    k = rms_norm(heads_view(linear(p, pre + ".attn.to_k", xn)), p[pre + ".attn.norm_k.weight"])
    v = heads_view(linear(p, pre + ".attn.to_v", xn))
    cq = rms_norm(heads_view(linear(p, pre + ".attn.add_q_proj", cn)), p[pre + ".attn.norm_added_q.weight"])
    ck = rms_norm(heads_view(linear(p, pre + ".attn.add_k_proj", cn)), p[pre + ".attn.norm_added_k.weight"])
    cv = heads_view(linear(p, pre + ".attn.add_v_proj", cn))
    t = ctx.shape[1]
    o = joint_attention(torch.cat([cq, q], 1), torch.cat([ck, k], 1), torch.cat([cv, v], 1), cs, mask, heads)
    attn_x = linear(p, pre + ".attn.to_out.0", o[:, t:])
    attn_c = linear(p, pre + ".attn.to_add_out", o[:, :t])

    x = x + g_a[:, None] * attn_x
    xn2 = layer_norm(x) * (1 + sc_m[:, None]) + sh_m[:, None]
    ff = linear(p, pre + ".ff.net.2", F.gelu(linear(p, pre + ".ff.net.0.proj", xn2), approximate="tanh"))
    x = x + g_m[:, None] * ff

    ctx = ctx + cg_a[:, None] * attn_c
    cn2 = layer_norm(ctx) * (1 + csc_m[:, None]) + csh_m[:, None]
    cff = linear(p, pre + ".ff_context.net.2", F.gelu(linear(p, pre + ".ff_context.net.0.proj", cn2), approximate="tanh"))
    ctx = ctx + cg_m[:, None] * cff
    return ctx, x


def single_block(p: Params, pre: str, x, temb, cs, mask, heads):
    """FluxSingleTransformerBlock.forward (B:914-942) + AdaLayerNormZeroSingle (N:217-249) + FluxSingleAttnProcessor2_0
    (B:745-785)."""
    b, s, d = x.shape
    hd = d // heads
    sh, sc, g = linear(p, pre + ".norm.linear", F.silu(temb)).chunk(3, dim=1)
    xn = layer_norm(x) * (1 + sc[:, None]) + sh[:, None]
    mlp = F.gelu(linear(p, pre + ".proj_mlp", xn), approximate="tanh")
    q = rms_norm(linear(p, pre + ".attn.to_q", xn).view(b, s, heads, hd), p[pre + ".attn.norm_q.weight"])
    k = rms_norm(linear(p, pre + ".attn.to_k", xn).view(b, s, heads, hd), p[pre + ".attn.norm_k.weight"])
    v = linear(p, pre + ".attn.to_v", xn).view(b, s, heads, hd)
    o = joint_attention(q, k, v, cs, mask, heads)
    out = linear(p, pre + ".proj_out", torch.cat([o, mlp], dim=2))
    return x + g[:, None] * out


# ------------------------------------------------------------------------------------------------------------------
# the full step
# ------------------------------------------------------------------------------------------------------------------
def patchify(clip: torch.Tensor, patch: int = 2) -> torch.Tensor:
    """'b c t h w -> b (t h w) (p1 p2 c)' (F:285-286)."""
    b, c, t, h, w = clip.shape
    x = clip.permute(0, 2, 3, 4, 1).reshape(b, t, h // patch, patch, w // patch, patch, c)
    return x.permute(0, 1, 2, 4, 3, 5, 6).reshape(b, t * (h // patch) * (w // patch), patch * patch * c)


def unpatchify(x: torch.Tensor, t: int, h: int, w: int, patch: int = 2) -> torch.Tensor:
    """split_output's reshape (F:383-387): [B, t*h*w, p*p*c] -> [B, c, t, h*p, w*p]."""
    b = x.shape[0]
    c = x.shape[-1] // (patch * patch)
    x = x.reshape(b, t, h, w, patch, patch, c).permute(0, 1, 2, 4, 3, 5, 6).reshape(b, t, h * patch, w * patch, c)
    return x.permute(0, 4, 1, 2, 3)


def flux_forward(p: Params, cfg: FluxConfig, clips: List[torch.Tensor], timestep: torch.Tensor,
                 encoder_hidden_states: torch.Tensor, encoder_attention_mask: torch.Tensor,
                 pooled_projections: torch.Tensor, return_intermediates: bool = False):
    """PyramidFluxTransformer.forward (F:392-542) for `sample=[clips]`; returns [B, C_lat, t, h, w] of the LAST clip."""
    dev = encoder_hidden_states.device
    heads = cfg.num_attention_heads
    temb = time_text_embed(p, timestep, pooled_projections)                     # F:400
    ctx = linear(p, "context_embedder", encoder_hidden_states)                  # F:401
    t_len = ctx.shape[1]
    tokens = torch.cat([patchify(c, cfg.patch_size) for c in clips], dim=1)      # F:281-289
    x = linear(p, "x_embedder", tokens)                                         # F:290
    ids = sequence_ids([c.shape for c in clips], t_len, cfg.patch_size)          # F:266-269
    cs = rope_table(ids, cfg.axes_dims_rope).to(dev)                             # F:270
    seg = token_segments(encoder_attention_mask, x.shape[1])                     # F:318-330
    mask = attention_mask(seg, ids[:, 0]).to(dev)                                # F:341-349
    inter = {}
    for i in range(cfg.num_layers):                                             # F:430-461
        ctx, x = double_block(p, f"transformer_blocks.{i}", x, ctx, temb, cs, mask, heads)
        if return_intermediates:
            inter[f"double{i}"] = torch.cat([ctx, x], 1).float().cpu()
    h = torch.cat([ctx, x], dim=1)                                              # F:463-489
    for i in range(cfg.num_single_layers):                                      # F:491-520
        h = single_block(p, f"single_transformer_blocks.{i}", h, temb, cs, mask, heads)
        if return_intermediates:
            inter[f"single{i}"] = h.float().cpu()
    h = h[:, t_len:]                                                            # F:529
    scale, shift = linear(p, "norm_out.linear", F.silu(temb).to(h.dtype)).chunk(2, dim=1)   # N:107-130 (scale first)
    h = layer_norm(h) * (1 + scale[:, None]) + shift[:, None]
    h = linear(p, "proj_out", h)                                                # F:539
    _, _, t, hh, ww = clips[-1].shape
    n_last = t * (hh // cfg.patch_size) * (ww // cfg.patch_size)
    out = unpatchify(h[:, -n_last:], t, hh // cfg.patch_size, ww // cfg.patch_size, cfg.patch_size)   # F:380-387
    if return_intermediates:
        return out, inter
    return out


# ------------------------------------------------------------------------------------------------------------------
# deterministic synthetic parameters (shared by golden generation, tests, bench)
# ------------------------------------------------------------------------------------------------------------------
def flux_param_shapes(cfg: FluxConfig) -> Dict[str, tuple]:
    """State-dict keys and shapes of PyramidFluxTransformer (verified against the reference by tests/golden)."""
    d = cfg.inner_dim
    hd = cfg.attention_head_dim
    s: Dict[str, tuple] = {}

    def lin(name, out_f, in_f):
        s[name + ".weight"] = (out_f, in_f)
        s[name + ".bias"] = (out_f,)

    lin("time_text_embed.timestep_embedder.linear_1", d, 256)
    lin("time_text_embed.timestep_embedder.linear_2", d, d)
    lin("time_text_embed.text_embedder.linear_1", d, cfg.pooled_projection_dim)
    lin("time_text_embed.text_embedder.linear_2", d, d)
    lin("context_embedder", d, cfg.joint_attention_dim)
    lin("x_embedder", d, cfg.in_channels)
    for i in range(cfg.num_layers):
        pre = f"transformer_blocks.{i}"
        lin(pre + ".norm1.linear", 6 * d, d)
        lin(pre + ".norm1_context.linear", 6 * d, d)
        for n in ("norm_q", "norm_k"):
            s[f"{pre}.attn.{n}.weight"] = (hd,)
        for n in ("to_q", "to_k", "to_v", "add_k_proj", "add_v_proj", "add_q_proj"):
            lin(f"{pre}.attn.{n}", d, d)
        lin(pre + ".attn.to_out.0", d, d)
        lin(pre + ".attn.to_add_out", d, d)
        for n in ("norm_added_q", "norm_added_k"):
            s[f"{pre}.attn.{n}.weight"] = (hd,)
        lin(pre + ".ff.net.0.proj", 4 * d, d)
        lin(pre + ".ff.net.2", d, 4 * d)
        lin(pre + ".ff_context.net.0.proj", 4 * d, d)
        lin(pre + ".ff_context.net.2", d, 4 * d)
    for i in range(cfg.num_single_layers):
        pre = f"single_transformer_blocks.{i}"
        lin(pre + ".norm.linear", 3 * d, d)
        lin(pre + ".proj_mlp", 4 * d, d)
        lin(pre + ".proj_out", d, 5 * d)
        for n in ("norm_q", "norm_k"):
            s[f"{pre}.attn.{n}.weight"] = (hd,)
        for n in ("to_q", "to_k", "to_v"):
            lin(f"{pre}.attn.{n}", d, d)
    lin("norm_out.linear", 2 * d, d)
    lin("proj_out", cfg.patch_size * cfg.patch_size * (cfg.in_channels // 4), d)
    return s


def synthetic_flux_params(cfg: FluxConfig, seed: int = 0, device: str = "cpu", bf16_representable: bool = True) -> Params:
    """Seeded non-degenerate parameters (the reference's own init zeroes AdaLN/proj_out => exactly-zero output,
    F:168-183).  Matrices ~ N(0, s^2) with s scaled so activations stay O(1) through 24 blocks; biases N(0, 0.02^2);
    norm weights 1 + N(0, 0.1^2).  With bf16_representable the matrices are rounded to bf16 values (kept in fp32) so the
    oracle and the bf16 CUDA path consume identical numbers."""
    g = torch.Generator().manual_seed(seed)
    out: Params = {}
    for name, shp in flux_param_shapes(cfg).items():
        if len(shp) == 2:
            fan_in = shp[1]
            std = 1.0 / math.sqrt(fan_in)
            if ".norm" in name and name.endswith("linear.weight"):
                std *= 0.5  # modulation (shift/scale/gate) ~ O(0.5)
            w = torch.randn(shp, generator=g) * std
            if bf16_representable:
                w = w.bfloat16().float()
            out[name] = w.to(device)
        elif name.endswith("weight"):
            out[name] = (1.0 + 0.1 * torch.randn(shp, generator=g)).to(device)
        else:
            out[name] = (0.02 * torch.randn(shp, generator=g)).to(device)
    return out
