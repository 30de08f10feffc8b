"""The prompt encoders of the pipeline on libpf_b200: T5 v1.1 encoder (T5-XXL) and the CLIP text transformer (CLIP-L, CLIP-G).

`B200FluxTextEncoder` and `B200SD3TextEncoder` replace the reference wrappers `FluxTextEncoderWithMask`
(pyramid_dit/flux_modules/modeling_text_encoder.py) and `SD3TextEncoderWithMask` (pyramid_dit/mmdit_modules/
modeling_text_encoder.py): same tokenizers, same padding and truncation, same three outputs, every matrix product, norm,
attention and activation on the library's sm_90a kernels (include/pf_b200.h "text encoders").  Launches per layer:
  T5 block:  RMSNorm, QKV GEMM, attention (relative position bias + key mask), O GEMM + residual, RMSNorm,
             GEGLU GEMM (wi_0 | wi_1 interleaved), wo GEMM + residual                                       (7)
  CLIP layer: LayerNorm, QKV GEMM + bias, causal attention, out_proj + residual, LayerNorm, fc1 + activation,
             fc2 + residual                                                                                 (7)
The residual streams are fp32; GEMM operands and outputs are bf16.  There is no CPU path: a forward with the weights on
the CPU raises.  `.to("cpu")` / `.to("cuda")` move the weights (they are buffers), which is what the pipeline's
cpu_offloading=True path does between calls.
"""
from __future__ import annotations

from typing import List, Optional, Union

import torch
import torch.nn as nn

from . import _lib, ops
from ._lib import (PF_EPI_GATE_RESID, PF_EPI_GEGLU_BF16, PF_EPI_GELU_BF16, PF_EPI_GELU_ERF_BF16, PF_EPI_QUICK_GELU_BF16,
                   PF_EPI_STORE_BF16)

T5_MAX_LENGTH = 128                    # the wrappers' _get_t5_prompt_embeds(max_sequence_length=128)
CLIP_ACT_EPILOGUE = {"quick_gelu": PF_EPI_QUICK_GELU_BF16, "gelu": PF_EPI_GELU_ERF_BF16,
                     "gelu_new": PF_EPI_GELU_BF16, "gelu_pytorch_tanh": PF_EPI_GELU_BF16}
T5_GATED_ACTS = ("gelu_new", "gelu_pytorch_tanh")    # GEGLU's gate is the tanh GELU


def interleave_geglu(wi_0: torch.Tensor, wi_1: torch.Tensor) -> torch.Tensor:
    """[d_ff, d] x 2 -> [2 d_ff, d]: 64-row blocks of wi_0 (gate) and wi_1 (linear) alternate, so that every 128-row block
    holds a gate block followed by its linear block (PF_EPI_GEGLU_BF16)."""
    f, d = wi_0.shape
    if f % 64 != 0 or wi_1.shape != wi_0.shape:
        raise ValueError(f"GEGLU weights must be two [d_ff, d] matrices with d_ff % 64 == 0 (got {tuple(wi_0.shape)}, "
                         f"{tuple(wi_1.shape)})")
    return torch.stack([wi_0.reshape(f // 64, 64, d), wi_1.reshape(f // 64, 64, d)], 1).reshape(2 * f, d)


def deinterleave_geglu(w: torch.Tensor):
    """Inverse of interleave_geglu."""
    f2, d = w.shape
    v = w.reshape(f2 // 128, 2, 64, d)
    return v[:, 0].reshape(f2 // 2, d), v[:, 1].reshape(f2 // 2, d)


def relative_position_bucket(relative_position: torch.Tensor, num_buckets: int, max_distance: int) -> torch.Tensor:
    """T5Attention._relative_position_bucket for the (bidirectional) encoder, with the same torch ops, so the buckets are
    exact."""
    import math
    num_buckets //= 2
    buckets = (relative_position > 0).to(torch.long) * num_buckets
    relative_position = torch.abs(relative_position)
    max_exact = num_buckets // 2
    is_small = relative_position < max_exact
    large = max_exact + (torch.log(relative_position.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return buckets + torch.where(is_small, relative_position, large)


def t5_bias_table(rel_bias_weight: torch.Tensor, seq: int, num_buckets: int, max_distance: int) -> torch.Tensor:
    """T5Attention.compute_bias(seq, seq) as the Toeplitz table of pf_attn_fwd_text: fp32 [heads, 2 seq - 1], entry
    k - q + seq - 1 = bias of (query q, key k)."""
    rel = torch.arange(-(seq - 1), seq, dtype=torch.long)
    bucket = relative_position_bucket(rel, num_buckets, max_distance)
    return rel_bias_weight.detach().float().cpu()[bucket].t().contiguous()


def clip_pooled_index(ids: torch.Tensor, eos_token_id: int) -> torch.Tensor:
    """The pooled row of CLIPTextTransformer.forward from the host copy of the ids: the argmax of the ids when
    eos_token_id == 2 (the legacy rule, which the released CLIP-L config takes), else the first position of eos_token_id."""
    ids = ids.to(torch.int)
    if eos_token_id == 2:
        return ids.argmax(dim=-1)
    return (ids == eos_token_id).int().argmax(dim=-1)


def _to_device(t: torch.Tensor, device) -> torch.Tensor:
    """Host -> device copy that does not wait for the kernels already queued on the stream (a copy from pageable memory
    would), so the second encoder of a wrapper is enqueued while the first one runs."""
    return t.contiguous().pin_memory().to(device, non_blocking=True)


def _cfg(config, name, default=None):
    v = getattr(config, name, default)
    return default if v is None else v


def _check_ids(ids: torch.Tensor, vocab: int, what: str) -> torch.Tensor:
    ids = ids.detach().to("cpu", torch.int64)
    if ids.dim() != 2 or ids.numel() == 0:
        raise ValueError(f"{what}: token ids must be a non-empty [batch, seq] tensor (got {tuple(ids.shape)})")
    lo, hi = int(ids.min()), int(ids.max())
    if lo < 0 or hi >= vocab:
        raise ValueError(f"{what}: token id out of range [0, {vocab}) (min {lo}, max {hi})")
    return ids


class _Encoder(nn.Module):
    """Weights as buffers on one device; the forward runs where they are and refuses the CPU."""

    def _bf16(self, t: torch.Tensor, device) -> torch.Tensor:
        return t.detach().float().to(device=device, dtype=torch.bfloat16).contiguous()

    def _f32(self, t: torch.Tensor, device) -> torch.Tensor:
        return t.detach().float().to(device=device).contiguous()

    @property
    def device(self) -> torch.device:
        return self.ones_gate.device

    @property
    def dtype(self) -> torch.dtype:
        return torch.bfloat16

    def _require_gpu(self, what: str) -> None:
        if self.device.type != "cuda":
            raise RuntimeError(f"{what}: the weights are on {self.device}; libpf_b200 has no CPU path (move the encoder "
                               "with .to('cuda') first)")
        _lib.require_device()


class B200T5Encoder(_Encoder):
    """T5EncoderModel.forward()[0] (T5 v1.1: gated GELU feed-forward, relative position bias from block 0, no biases)."""

    def __init__(self, config, state_dict, device="cuda"):
        super().__init__()
        self.d_model, self.heads, self.d_kv = int(config.d_model), int(config.num_heads), int(config.d_kv)
        self.num_layers, self.d_ff, self.vocab = int(config.num_layers), int(config.d_ff), int(config.vocab_size)
        self.num_buckets = int(_cfg(config, "relative_attention_num_buckets", 32))
        self.max_distance = int(_cfg(config, "relative_attention_max_distance", 128))
        self.eps = float(_cfg(config, "layer_norm_epsilon", 1e-6))
        act = _cfg(config, "dense_act_fn", None) or _cfg(config, "hidden_act", "gelu_new")
        if not bool(_cfg(config, "is_gated_act", False)):
            raise ValueError("B200T5Encoder supports the gated feed-forward of T5 v1.1 only (is_gated_act=False given)")
        if act not in T5_GATED_ACTS:
            raise ValueError(f"B200T5Encoder: dense_act_fn {act!r} unsupported (one of {T5_GATED_ACTS})")
        if self.d_kv != 64:
            raise ValueError(f"B200T5Encoder: head_dim (d_kv) {self.d_kv} unsupported (64 only)")
        dev = torch.device(device)
        sd = state_dict
        reg = self.register_buffer
        reg("embed", self._bf16(sd["shared.weight"], dev))
        self.rel_bias = sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"].detach().float().cpu()
        reg("ones_gate", torch.ones(self.d_model, device=dev, dtype=torch.float32))
        for i in range(self.num_layers):
            p = f"encoder.block.{i}.layer."
            reg(f"l{i}_ln0", self._f32(sd[p + "0.layer_norm.weight"], dev))
            reg(f"l{i}_qkv", self._bf16(torch.cat([sd[p + f"0.SelfAttention.{n}.weight"].float() for n in "qkv"], 0), dev))
            reg(f"l{i}_o", self._bf16(sd[p + "0.SelfAttention.o.weight"], dev))
            reg(f"l{i}_ln1", self._f32(sd[p + "1.layer_norm.weight"], dev))
            reg(f"l{i}_wi", self._bf16(interleave_geglu(sd[p + "1.DenseReluDense.wi_0.weight"].float(),
                                                        sd[p + "1.DenseReluDense.wi_1.weight"].float()), dev))
            reg(f"l{i}_wo", self._bf16(sd[p + "1.DenseReluDense.wo.weight"], dev))
        reg("ln_f", self._f32(sd["encoder.final_layer_norm.weight"], dev))
        self._bias_tables = {}

    def bias_table(self, seq: int) -> torch.Tensor:
        """The relative position bias of `seq` tokens, built once per (seq, device); every layer shares it."""
        key = (seq, self.device)
        if key not in self._bias_tables:
            self._bias_tables[key] = t5_bias_table(self.rel_bias, seq, self.num_buckets, self.max_distance).to(self.device)
        return self._bias_tables[key]

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
        """input_ids [B, S], attention_mask {0, 1} [B, S] -> last_hidden_state bf16 [B, S, d_model]."""
        ids = _check_ids(input_ids, self.vocab, "B200T5Encoder")
        b, s = ids.shape
        mask = attention_mask.detach().to("cpu", torch.int32)
        if tuple(mask.shape) != (b, s):
            raise ValueError(f"B200T5Encoder: attention_mask {tuple(mask.shape)} does not match the ids {(b, s)}")
        if bool((mask.sum(1) == 0).any()):
            raise ValueError("B200T5Encoder: a sequence whose attention mask is all zeros has no key to attend to")
        self._require_gpu("B200T5Encoder")
        dev, d, inner, m = self.device, self.d_model, self.heads * self.d_kv, b * s
        ids_d = _to_device(ids.to(torch.int32).reshape(-1), dev)
        mask_d = _to_device(mask, dev)
        bias = self.bias_table(s)
        x = torch.empty(m, d, device=dev, dtype=torch.float32)
        h = torch.empty(m, d, device=dev, dtype=torch.bfloat16)
        qkv = torch.empty(m, 3 * inner, device=dev, dtype=torch.bfloat16)
        att = torch.empty(m, inner, device=dev, dtype=torch.bfloat16)
        ff = torch.empty(m, self.d_ff, device=dev, dtype=torch.bfloat16)
        ops.embed_tokens(ids_d, self.embed, x, rows_per_batch=s)
        resid = dict(rows_per_batch=m, out=x, gate=self.ones_gate)
        for i in range(self.num_layers):
            ops.rms_norm_rows(x, h, getattr(self, f"l{i}_ln0"), eps=self.eps)
            ops.gemm(h, getattr(self, f"l{i}_qkv"), None, PF_EPI_STORE_BF16, rows_per_batch=m, out=qkv)
            ops.attn_fwd_text(qkv, att, batch=b, heads=self.heads, seq=s, scale=1.0, bias=bias, key_mask=mask_d)
            ops.gemm(att, getattr(self, f"l{i}_o"), None, PF_EPI_GATE_RESID, **resid)
            ops.rms_norm_rows(x, h, getattr(self, f"l{i}_ln1"), eps=self.eps)
            ops.gemm(h, getattr(self, f"l{i}_wi"), None, PF_EPI_GEGLU_BF16, rows_per_batch=m, out=ff)
            ops.gemm(ff, getattr(self, f"l{i}_wo"), None, PF_EPI_GATE_RESID, **resid)
        ops.rms_norm_rows(x, h, self.ln_f, eps=self.eps)
        return h.view(b, s, d)


class B200CLIPText(_Encoder):
    """CLIPTextTransformer.forward's pooled output (+ CLIPTextModelWithProjection's text_projection when the state dict has
    one): causal self-attention, pre-LayerNorm layers, final_layer_norm applied to the pooled rows."""

    def __init__(self, config, state_dict, device="cuda"):
        super().__init__()
        self.hidden, self.heads = int(config.hidden_size), int(config.num_attention_heads)
        self.num_layers, self.vocab = int(config.num_hidden_layers), int(config.vocab_size)
        self.max_pos = int(config.max_position_embeddings)
        self.eos_token_id = int(config.eos_token_id)
        self.eps = float(_cfg(config, "layer_norm_eps", 1e-5))
        act = config.hidden_act
        if act not in CLIP_ACT_EPILOGUE:
            raise ValueError(f"B200CLIPText: hidden_act {act!r} unsupported (one of {tuple(CLIP_ACT_EPILOGUE)})")
        if self.hidden % self.heads != 0 or self.hidden // self.heads != 64:
            raise ValueError(f"B200CLIPText: head_dim {self.hidden / self.heads:g} unsupported (64 only)")
        self.act_epilogue = CLIP_ACT_EPILOGUE[act]
        dev = torch.device(device)
        sd, tm = state_dict, "text_model."
        reg = self.register_buffer
        reg("tok_embed", self._bf16(sd[tm + "embeddings.token_embedding.weight"], dev))
        reg("pos_embed", self._bf16(sd[tm + "embeddings.position_embedding.weight"], dev))
        reg("ones_gate", torch.ones(self.hidden, device=dev, dtype=torch.float32))

        def ln(name, key):   # LayerNorm as pf_ln_modulate: shift = bias, scale = weight - 1
            reg(key + "_shift", self._f32(sd[name + ".bias"], dev))
            reg(key + "_scale", self._f32(sd[name + ".weight"].float() - 1.0, dev))

        for i in range(self.num_layers):
            p = f"{tm}encoder.layers.{i}."
            ln(p + "layer_norm1", f"l{i}_ln1")
            ln(p + "layer_norm2", f"l{i}_ln2")
            names = [p + f"self_attn.{n}" for n in ("q_proj", "k_proj", "v_proj")]
            reg(f"l{i}_qkv", self._bf16(torch.cat([sd[n + ".weight"].float() for n in names], 0), dev))
            reg(f"l{i}_qkv_b", self._f32(torch.cat([sd[n + ".bias"].float() for n in names], 0), dev))
            for key, n in (("o", "self_attn.out_proj"), ("fc1", "mlp.fc1"), ("fc2", "mlp.fc2")):
                reg(f"l{i}_{key}", self._bf16(sd[p + n + ".weight"], dev))
                reg(f"l{i}_{key}_b", self._f32(sd[p + n + ".bias"], dev))
        ln(tm + "final_layer_norm", "ln_f")
        self.has_projection = "text_projection.weight" in sd
        if self.has_projection:
            reg("proj", self._bf16(sd["text_projection.weight"], dev))
        self.out_dim = int(sd["text_projection.weight"].shape[0]) if self.has_projection else self.hidden

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor) -> torch.Tensor:
        """input_ids [B, S] -> pooler_output bf16 [B, hidden], or text_embeds bf16 [B, projection_dim] with a projection."""
        ids = _check_ids(input_ids, self.vocab, "B200CLIPText")
        b, s = ids.shape
        if s > self.max_pos:
            raise ValueError(f"B200CLIPText: {s} tokens exceed max_position_embeddings {self.max_pos}")
        pooled_rows = clip_pooled_index(ids, self.eos_token_id) + torch.arange(b) * s
        self._require_gpu("B200CLIPText")
        dev, d, m = self.device, self.hidden, b * s
        x = torch.empty(m, d, device=dev, dtype=torch.float32)
        h = torch.empty(m, d, device=dev, dtype=torch.bfloat16)
        qkv = torch.empty(m, 3 * d, device=dev, dtype=torch.bfloat16)
        att = torch.empty(m, d, device=dev, dtype=torch.bfloat16)
        mlp = torch.empty(m, getattr(self, "l0_fc1").shape[0], device=dev, dtype=torch.bfloat16)
        ops.embed_tokens(_to_device(ids.to(torch.int32).reshape(-1), dev), self.tok_embed, x, rows_per_batch=s,
                         pos_table=self.pos_embed)
        rows = dict(batches=1, rows_per_batch=m, row_begin=0, row_count=m, eps=self.eps)
        for i in range(self.num_layers):
            g = lambda k: getattr(self, f"l{i}_{k}")  # noqa: E731
            ops.ln_modulate(x, h, g("ln1_shift"), g("ln1_scale"), 0, **rows)
            ops.gemm(h, g("qkv"), g("qkv_b"), PF_EPI_STORE_BF16, rows_per_batch=m, out=qkv)
            ops.attn_fwd_text(qkv, att, batch=b, heads=self.heads, seq=s, scale=0.125, causal=True)
            ops.gemm(att, g("o"), g("o_b"), PF_EPI_GATE_RESID, rows_per_batch=m, out=x, gate=self.ones_gate)
            ops.ln_modulate(x, h, g("ln2_shift"), g("ln2_scale"), 0, **rows)
            ops.gemm(h, g("fc1"), g("fc1_b"), self.act_epilogue, rows_per_batch=m, out=mlp)
            ops.gemm(mlp, g("fc2"), g("fc2_b"), PF_EPI_GATE_RESID, rows_per_batch=m, out=x, gate=self.ones_gate)
        # final_layer_norm of the pooled rows only (the other rows of last_hidden_state are not returned)
        xp = x.index_select(0, _to_device(pooled_rows, dev)).contiguous()
        pooled = torch.empty(b, d, device=dev, dtype=torch.bfloat16)
        ops.ln_modulate(xp, pooled, self.ln_f_shift, self.ln_f_scale, 0, batches=1, rows_per_batch=b, row_begin=0, row_count=b,
                        eps=self.eps)
        if not self.has_projection:
            return pooled
        out = torch.empty(b, self.out_dim, device=dev, dtype=torch.bfloat16)
        ops.gemm(pooled, self.proj, None, PF_EPI_STORE_BF16, rows_per_batch=b, out=out)
        return out


def _state_dict_and_config(hf_model):
    return hf_model.config, hf_model.state_dict()


class _TextEncoderWrapper(nn.Module):
    """Tokenisation exactly as the reference wrappers (padding="max_length", truncation), encoders on the library."""

    def _t5_tokens(self, tokenizer, prompts: List[str]):
        t = tokenizer(prompts, padding="max_length", max_length=T5_MAX_LENGTH, truncation=True, add_special_tokens=True,
                      return_tensors="pt")
        return t.input_ids, t.attention_mask

    def _clip_tokens(self, tokenizer, prompts: List[str]):
        return tokenizer(prompts, padding="max_length", max_length=self.tokenizer_max_length, truncation=True,
                         return_tensors="pt").input_ids

    @property
    def device(self) -> torch.device:
        return self.t5.device

    @property
    def dtype(self) -> torch.dtype:
        return torch.bfloat16


class B200FluxTextEncoder(_TextEncoderWrapper):
    """FluxTextEncoderWithMask on the library: CLIP-L pooled output + T5-XXL.  forward(prompts, device) ->
    (prompt_embeds bf16 [B, 128, 4096], prompt_attention_mask int64 [B, 128], pooled_prompt_embeds bf16 [B, 768])."""

    def __init__(self, tokenizer, tokenizer_2, clip: B200CLIPText, t5: B200T5Encoder, tokenizer_max_length: Optional[int] = None):
        super().__init__()
        self.tokenizer, self.tokenizer_2 = tokenizer, tokenizer_2
        self.tokenizer_max_length = tokenizer_max_length or (tokenizer.model_max_length if tokenizer is not None else 77)
        self.clip, self.t5 = clip, t5

    @classmethod
    def from_reference(cls, ref, device="cuda") -> "B200FluxTextEncoder":
        """From a FluxTextEncoderWithMask: its tokenizers and the weights of its two models (the HF models are not kept)."""
        c1, s1 = _state_dict_and_config(ref.text_encoder)
        c2, s2 = _state_dict_and_config(ref.text_encoder_2)
        return cls(ref.tokenizer, ref.tokenizer_2, B200CLIPText(c1, s1, device), B200T5Encoder(c2, s2, device),
                   tokenizer_max_length=ref.tokenizer_max_length)

    def encode_ids(self, clip_ids: torch.Tensor, t5_ids: torch.Tensor, t5_mask: torch.Tensor, device=None):
        pooled = self.clip(clip_ids)
        embeds = self.t5(t5_ids, t5_mask)
        device = self.device if device is None else device
        return embeds.to(device), _to_device(t5_mask.to(torch.int64), device), pooled.to(device)

    def forward(self, input_prompts: Union[str, List[str]], device):
        prompts = [input_prompts] if isinstance(input_prompts, str) else list(input_prompts)
        t5_ids, t5_mask = self._t5_tokens(self.tokenizer_2, prompts)
        return self.encode_ids(self._clip_tokens(self.tokenizer, prompts), t5_ids, t5_mask, device)


class B200SD3TextEncoder(_TextEncoderWrapper):
    """SD3TextEncoderWithMask on the library: CLIP-L and CLIP-G text_embeds (concatenated) + T5-XXL.  forward(prompts,
    device) -> (prompt_embeds bf16 [B, 128, 4096], prompt_attention_mask int64 [B, 128], pooled_prompt_embeds bf16 [B, 2048])."""

    def __init__(self, tokenizer, tokenizer_2, tokenizer_3, clip_l: B200CLIPText, clip_g: B200CLIPText, t5: B200T5Encoder,
                 tokenizer_max_length: Optional[int] = None):
        super().__init__()
        self.tokenizer, self.tokenizer_2, self.tokenizer_3 = tokenizer, tokenizer_2, tokenizer_3
        self.tokenizer_max_length = tokenizer_max_length or tokenizer.model_max_length
        self.clip_l, self.clip_g, self.t5 = clip_l, clip_g, t5

    @classmethod
    def from_reference(cls, ref, device="cuda") -> "B200SD3TextEncoder":
        """From an SD3TextEncoderWithMask: its three tokenizers and the weights of its three models."""
        enc = [B200CLIPText(*_state_dict_and_config(ref.text_encoder), device),
               B200CLIPText(*_state_dict_and_config(ref.text_encoder_2), device),
               B200T5Encoder(*_state_dict_and_config(ref.text_encoder_3), device)]
        return cls(ref.tokenizer, ref.tokenizer_2, ref.tokenizer_3, *enc, tokenizer_max_length=ref.tokenizer_max_length)

    def encode_ids(self, clip_l_ids: torch.Tensor, clip_g_ids: torch.Tensor, t5_ids: torch.Tensor, t5_mask: torch.Tensor,
                   device=None):
        pooled = torch.cat([self.clip_l(clip_l_ids), self.clip_g(clip_g_ids)], dim=-1)
        embeds = self.t5(t5_ids, t5_mask)
        device = self.device if device is None else device
        return embeds.to(device), _to_device(t5_mask.to(torch.int64), device), pooled.to(device)

    def forward(self, input_prompts: Union[str, List[str]], device):
        prompts = [input_prompts] if isinstance(input_prompts, str) else list(input_prompts)
        t5_ids, t5_mask = self._t5_tokens(self.tokenizer_3, prompts)
        return self.encode_ids(self._clip_tokens(self.tokenizer, prompts), self._clip_tokens(self.tokenizer_2, prompts),
                               t5_ids, t5_mask, device)
