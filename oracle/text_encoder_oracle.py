"""Restatement of the text encoders the pipeline runs, as pure functions over transformers' state-dict key layout.

TEST-ONLY: the golden tests (tests/test_text_encoder_*.py) compare the library against these functions, and
oracle/pin/make_text_golden.py pins them against the unmodified reference wrappers (FluxTextEncoderWithMask,
SD3TextEncoderWithMask) built on transformers' CLIPTextModel[WithProjection] / T5EncoderModel.

  * clip_text_forward  CLIPTextTransformer.forward (+ CLIPTextModelWithProjection's text_projection)
  * t5_encoder_forward T5EncoderModel.forward: T5Stack of T5Block (T5LayerSelfAttention, T5LayerFF with
                       T5DenseGatedActDense), relative position bias from block 0, T5LayerNorm, final_layer_norm

Both compute in the dtype of the parameters they are given: with fp32 parameters they are the fp32 reference, with the
parameters cast to bf16 they follow the casts transformers makes for a bf16 checkpoint (fp32 variance in T5LayerNorm, fp32
softmax, everything else in bf16), which is the reference's own bf16 numerics.  transformers keeps T5's `wo` in fp32 only
for fp16 loads (`_keep_in_fp32_modules`); for bf16 it is bf16 like every other weight, and so it is here.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch
import torch.nn.functional as F

Params = Dict[str, torch.Tensor]


@dataclass
class ClipTextConfig:
    vocab_size: int = 49408
    hidden_size: int = 768
    num_attention_heads: int = 12
    num_hidden_layers: int = 12
    intermediate_size: int = 3072
    max_position_embeddings: int = 77
    hidden_act: str = "quick_gelu"
    eos_token_id: int = 2
    layer_norm_eps: float = 1e-5
    projection_dim: Optional[int] = None   # CLIPTextModelWithProjection's text_projection (no bias) when set


@dataclass
class T5EncoderConfig:
    vocab_size: int = 32128
    d_model: int = 4096
    d_kv: int = 64
    num_heads: int = 64
    num_layers: int = 24
    d_ff: int = 10240
    relative_attention_num_buckets: int = 32
    relative_attention_max_distance: int = 128
    layer_norm_epsilon: float = 1e-6
    dense_act_fn: str = "gelu_new"
    is_gated_act: bool = True


# the released configurations (CLIP-L of FLUX.1 / SD3, CLIP-G of SD3, T5 v1.1 XXL)
CLIP_L = ClipTextConfig()
CLIP_L_PROJ = ClipTextConfig(projection_dim=768)
CLIP_G = ClipTextConfig(hidden_size=1280, num_attention_heads=20, num_hidden_layers=32, intermediate_size=5120,
                        hidden_act="gelu", eos_token_id=49407, projection_dim=1280)
T5_XXL = T5EncoderConfig()

_ACT = {
    "quick_gelu": lambda x: x * torch.sigmoid(1.702 * x),
    "gelu": lambda x: F.gelu(x),
    "gelu_new": lambda x: F.gelu(x, approximate="tanh"),
    "gelu_pytorch_tanh": lambda x: F.gelu(x, approximate="tanh"),
}


# ---- synthetic parameters (scales of CLIPPreTrainedModel._init_weights / T5PreTrainedModel._init_weights) ------------
def _randn(g, shape, std, device):
    return torch.randn(shape, generator=g, device=device) * std


def synthetic_clip_params(cfg: ClipTextConfig, seed: int = 0, device="cpu") -> Params:
    """Weights at the init scales; biases N(0, 0.02^2) and LayerNorm weights 1 + N(0, 0.05^2) (not the init's zeros / ones) so
    that every parameter is exercised."""
    g = torch.Generator(device=device).manual_seed(seed)
    d, f, n = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers
    in_std = d ** -0.5 * (2 * n) ** -0.5
    p: Params = {
        "text_model.embeddings.token_embedding.weight": _randn(g, (cfg.vocab_size, d), 0.02, device),
        "text_model.embeddings.position_embedding.weight": _randn(g, (cfg.max_position_embeddings, d), 0.02, device),
    }
    for i in range(n):
        pre = f"text_model.encoder.layers.{i}."
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            p[pre + f"self_attn.{nm}.weight"] = _randn(g, (d, d), d ** -0.5 if nm == "out_proj" else in_std, device)
            p[pre + f"self_attn.{nm}.bias"] = _randn(g, (d,), 0.02, device)
        for ln in ("layer_norm1", "layer_norm2"):
            p[pre + f"{ln}.weight"] = 1.0 + _randn(g, (d,), 0.05, device)
            p[pre + f"{ln}.bias"] = _randn(g, (d,), 0.02, device)
        p[pre + "mlp.fc1.weight"] = _randn(g, (f, d), (2 * d) ** -0.5, device)
        p[pre + "mlp.fc1.bias"] = _randn(g, (f,), 0.02, device)
        p[pre + "mlp.fc2.weight"] = _randn(g, (d, f), in_std, device)
        p[pre + "mlp.fc2.bias"] = _randn(g, (d,), 0.02, device)
    p["text_model.final_layer_norm.weight"] = 1.0 + _randn(g, (d,), 0.05, device)
    p["text_model.final_layer_norm.bias"] = _randn(g, (d,), 0.02, device)
    if cfg.projection_dim is not None:
        p["text_projection.weight"] = _randn(g, (cfg.projection_dim, d), d ** -0.5, device)
    return p


def synthetic_t5_params(cfg: T5EncoderConfig, seed: int = 0, device="cpu") -> Params:
    """Weights at the init scales; T5LayerNorm weights 1 + N(0, 0.05^2) (not the init's ones)."""
    g = torch.Generator(device=device).manual_seed(seed)
    d, inner, f = cfg.d_model, cfg.num_heads * cfg.d_kv, cfg.d_ff
    p: Params = {"shared.weight": _randn(g, (cfg.vocab_size, d), 1.0, device)}
    for i in range(cfg.num_layers):
        pre = f"encoder.block.{i}.layer."
        p[pre + "0.SelfAttention.q.weight"] = _randn(g, (inner, d), (d * cfg.d_kv) ** -0.5, device)
        p[pre + "0.SelfAttention.k.weight"] = _randn(g, (inner, d), d ** -0.5, device)
        p[pre + "0.SelfAttention.v.weight"] = _randn(g, (inner, d), d ** -0.5, device)
        p[pre + "0.SelfAttention.o.weight"] = _randn(g, (d, inner), inner ** -0.5, device)
        if i == 0:
            p[pre + "0.SelfAttention.relative_attention_bias.weight"] = _randn(
                g, (cfg.relative_attention_num_buckets, cfg.num_heads), d ** -0.5, device)
        p[pre + "0.layer_norm.weight"] = 1.0 + _randn(g, (d,), 0.05, device)
        p[pre + "1.DenseReluDense.wi_0.weight"] = _randn(g, (f, d), d ** -0.5, device)
        p[pre + "1.DenseReluDense.wi_1.weight"] = _randn(g, (f, d), d ** -0.5, device)
        p[pre + "1.DenseReluDense.wo.weight"] = _randn(g, (d, f), f ** -0.5, device)
        p[pre + "1.layer_norm.weight"] = 1.0 + _randn(g, (d,), 0.05, device)
    p["encoder.final_layer_norm.weight"] = 1.0 + _randn(g, (d,), 0.05, device)
    return p


# ---- CLIP text -------------------------------------------------------------------------------------------------------
def clip_eos_index(ids: torch.Tensor, eos_token_id: int) -> torch.Tensor:
    """Pooled row of CLIPTextTransformer.forward: the legacy argmax of the ids when eos_token_id == 2, else the first
    position holding eos_token_id."""
    if eos_token_id == 2:
        return ids.to(torch.int).argmax(dim=-1)
    return (ids.to(torch.int) == eos_token_id).int().argmax(dim=-1)


def clip_text_forward(p: Params, cfg: ClipTextConfig, ids: torch.Tensor):
    """ids int [B, S] -> (last_hidden_state [B, S, d], pooler_output [B, d], text_embeds [B, proj] or None)."""
    tm = "text_model."
    b, s = ids.shape
    d, nh = cfg.hidden_size, cfg.num_attention_heads
    hd = d // nh
    x = p[tm + "embeddings.token_embedding.weight"][ids] + p[tm + "embeddings.position_embedding.weight"][:s][None]
    dt = x.dtype
    causal = torch.full((s, s), torch.finfo(dt).min, dtype=dt, device=x.device).triu(1)
    act = _ACT[cfg.hidden_act]

    def ln(v, name):
        return F.layer_norm(v, (d,), p[name + ".weight"], p[name + ".bias"], cfg.layer_norm_eps)

    def lin(v, name, bias=True):
        return F.linear(v, p[name + ".weight"], p[name + ".bias"] if bias else None)

    for i in range(cfg.num_hidden_layers):
        pre = f"{tm}encoder.layers.{i}."
        h = ln(x, pre + "layer_norm1")
        q, k, v = (lin(h, pre + f"self_attn.{n}").view(b, s, nh, hd).transpose(1, 2) for n in ("q_proj", "k_proj", "v_proj"))
        w = torch.matmul(q, k.transpose(-1, -2)) * hd ** -0.5 + causal
        w = torch.softmax(w, dim=-1, dtype=torch.float32).to(dt)
        a = torch.matmul(w, v).transpose(1, 2).reshape(b, s, d)
        x = x + lin(a, pre + "self_attn.out_proj")
        h = ln(x, pre + "layer_norm2")
        x = x + lin(act(lin(h, pre + "mlp.fc1")), pre + "mlp.fc2")
    last = ln(x, tm + "final_layer_norm")
    pooled = last[torch.arange(b, device=last.device), clip_eos_index(ids, cfg.eos_token_id).to(last.device)]
    text_embeds = F.linear(pooled, p["text_projection.weight"]) if cfg.projection_dim is not None else None
    return last, pooled, text_embeds


# ---- T5 encoder ------------------------------------------------------------------------------------------------------
def relative_position_bucket(relative_position: torch.Tensor, num_buckets: int, max_distance: int) -> torch.Tensor:
    """T5Attention._relative_position_bucket, bidirectional (the encoder), the same torch ops."""
    num_buckets //= 2
    buckets = (relative_position > 0).to(torch.long) * num_buckets
    relative_position = torch.abs(relative_position)
    max_exact = num_buckets // 2
    is_small = relative_position < max_exact
    large = max_exact + (torch.log(relative_position.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return buckets + torch.where(is_small, relative_position, large)


def t5_position_bias(rel_bias_weight: torch.Tensor, cfg: T5EncoderConfig, seq: int) -> torch.Tensor:
    """T5Attention.compute_bias(seq, seq): [1, heads, seq, seq] in the dtype of the bias table."""
    pos = torch.arange(seq, dtype=torch.long, device=rel_bias_weight.device)
    rel = pos[None, :] - pos[:, None]
    bucket = relative_position_bucket(rel, cfg.relative_attention_num_buckets, cfg.relative_attention_max_distance)
    return F.embedding(bucket, rel_bias_weight).permute(2, 0, 1).unsqueeze(0)


def t5_layer_norm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    var = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
    x = x * torch.rsqrt(var + eps)
    if w.dtype in (torch.float16, torch.bfloat16):
        x = x.to(w.dtype)
    return w * x


def t5_encoder_forward(p: Params, cfg: T5EncoderConfig, ids: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """ids int [B, S], mask {0, 1} [B, S] -> last_hidden_state [B, S, d_model] (T5EncoderModel.forward()[0])."""
    b, s = ids.shape
    nh, hd = cfg.num_heads, cfg.d_kv
    x = p["shared.weight"][ids]
    dt = x.dtype
    ext = (1.0 - mask.to(dt))[:, None, None, :] * torch.finfo(dt).min    # the T5Stack additive key mask
    bias = t5_position_bias(p["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"], cfg, s) + ext
    act = _ACT[cfg.dense_act_fn]
    eps = cfg.layer_norm_epsilon
    for i in range(cfg.num_layers):
        pre = f"encoder.block.{i}.layer."
        h = t5_layer_norm(x, p[pre + "0.layer_norm.weight"], eps)
        q, k, v = (F.linear(h, p[pre + f"0.SelfAttention.{n}.weight"]).view(b, s, nh, hd).transpose(1, 2) for n in "qkv")
        sc = torch.matmul(q, k.transpose(3, 2)) + bias
        w = torch.softmax(sc.float(), dim=-1).type_as(sc)
        a = torch.matmul(w, v).transpose(1, 2).reshape(b, s, nh * hd)
        x = x + F.linear(a, p[pre + "0.SelfAttention.o.weight"])
        h = t5_layer_norm(x, p[pre + "1.layer_norm.weight"], eps)
        ff = act(F.linear(h, p[pre + "1.DenseReluDense.wi_0.weight"])) * F.linear(h, p[pre + "1.DenseReluDense.wi_1.weight"])
        x = x + F.linear(ff, p[pre + "1.DenseReluDense.wo.weight"])
    return t5_layer_norm(x, p["encoder.final_layer_norm.weight"], eps)


def to_dtype(p: Params, dtype: torch.dtype) -> Params:
    return {k: v.to(dtype) for k, v in p.items()}


# ---- transformers models and tokenizers of a given configuration (pinning script and drop-in tests) -------------------
def hf_clip_config(cfg: ClipTextConfig):
    from transformers import CLIPTextConfig
    kw = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
              num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
              max_position_embeddings=cfg.max_position_embeddings, hidden_act=cfg.hidden_act, eos_token_id=cfg.eos_token_id,
              layer_norm_eps=cfg.layer_norm_eps, attention_dropout=0.0)
    if cfg.projection_dim is not None:
        kw["projection_dim"] = cfg.projection_dim
    return CLIPTextConfig(**kw)


def hf_t5_config(cfg: T5EncoderConfig):
    from transformers import T5Config
    return T5Config(vocab_size=cfg.vocab_size, d_model=cfg.d_model, d_kv=cfg.d_kv, d_ff=cfg.d_ff, num_layers=cfg.num_layers,
                    num_heads=cfg.num_heads, relative_attention_num_buckets=cfg.relative_attention_num_buckets,
                    relative_attention_max_distance=cfg.relative_attention_max_distance, dropout_rate=0.0,
                    layer_norm_epsilon=cfg.layer_norm_epsilon, feed_forward_proj="gated-gelu", is_encoder_decoder=False,
                    use_cache=False)


def hf_clip_model(cfg: ClipTextConfig, params: Params):
    from transformers import CLIPTextModel, CLIPTextModelWithProjection
    cls = CLIPTextModel if cfg.projection_dim is None else CLIPTextModelWithProjection
    m = cls(hf_clip_config(cfg)).eval()
    m.load_state_dict(params, strict=True)
    return m


def hf_t5_model(cfg: T5EncoderConfig, params: Params):
    from transformers import T5EncoderModel
    m = T5EncoderModel(hf_t5_config(cfg)).eval()
    sd = dict(params)
    sd["encoder.embed_tokens.weight"] = params["shared.weight"]     # tied to `shared` in T5EncoderModel
    m.load_state_dict(sd, strict=True)
    return m


def clip_tokenizer(vocab: Dict[str, int], merges, model_max_length: int = 77):
    """A byte-level BPE CLIPTokenizer from its vocab.json / merges.txt contents (pad token = <|endoftext|>)."""
    import json
    import os
    import tempfile
    from transformers import CLIPTokenizer
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "vocab.json"), "w") as f:
            json.dump(vocab, f)
        with open(os.path.join(d, "merges.txt"), "w") as f:
            f.write("#version: 0.2\n" + "\n".join(merges) + "\n")
        return CLIPTokenizer(os.path.join(d, "vocab.json"), os.path.join(d, "merges.txt"), model_max_length=model_max_length,
                             pad_token="<|endoftext|>")


def t5_tokenizer(tokenizer_json: str):
    """T5TokenizerFast around an in-memory `tokenizers` model (serialised with Tokenizer.to_str())."""
    from tokenizers import Tokenizer
    from transformers import T5TokenizerFast
    return T5TokenizerFast(tokenizer_object=Tokenizer.from_str(tokenizer_json), eos_token="</s>", pad_token="<pad>",
                           unk_token="<unk>", extra_ids=0)
