"""Text encoders without a GPU: the oracle against the reference wrappers' outputs (tests/golden/text_encoder_small.pt), the
T5 bias table, the GEGLU weight layout, the CLIP pooled-row rules, the configurations and inputs B200T5Encoder /
B200CLIPText refuse, and the validation of the new C-ABI entry points."""
import ctypes as C

import pytest
import torch

from oracle import text_encoder_oracle as TO
from pyramid_flow_b200 import _lib
from pyramid_flow_b200.text_encoder import (B200CLIPText, B200T5Encoder, clip_pooled_index, deinterleave_geglu,
                                            interleave_geglu, t5_bias_table)


def _golden(golden_dir):
    g = torch.load(golden_dir / "text_encoder_small.pt", weights_only=False)
    cfgs = {k: (TO.ClipTextConfig if k.split("_")[1] == "clip" else TO.T5EncoderConfig)(**v) for k, v in g["configs"].items()}
    params = {k: (TO.synthetic_clip_params if isinstance(c, TO.ClipTextConfig) else TO.synthetic_t5_params)(c, g["seeds"][k])
              for k, c in cfgs.items()}
    return g, cfgs, params


def test_oracle_matches_reference_wrappers(golden_dir):
    g, cfgs, p = _golden(golden_dir)
    with torch.no_grad():
        pooled = TO.clip_text_forward(p["flux_clip"], cfgs["flux_clip"], g["clip_ids"])[1]
        embeds = TO.t5_encoder_forward(p["flux_t5"], cfgs["flux_t5"], g["t5_ids"], g["t5_mask"])
        assert (pooled - g["flux"]["pooled_prompt_embeds"]).abs().max().item() < 1e-5
        assert (embeds - g["flux"]["prompt_embeds"]).abs().max().item() < 1e-5
        sd3_pooled = torch.cat([TO.clip_text_forward(p[k], cfgs[k], g["clip_ids"])[2] for k in ("sd3_clip_l", "sd3_clip_g")], -1)
        sd3_embeds = TO.t5_encoder_forward(p["sd3_t5"], cfgs["sd3_t5"], g["t5_ids"], g["t5_mask"])
        assert (sd3_pooled - g["sd3"]["pooled_prompt_embeds"]).abs().max().item() < 1e-5
        assert (sd3_embeds - g["sd3"]["prompt_embeds"]).abs().max().item() < 1e-5
    for name in ("flux", "sd3"):
        assert torch.equal(g[name]["prompt_attention_mask"], g["t5_mask"])
    # the fixture covers padded, unpadded and truncated prompts for both tokenizers
    t5_len = g["t5_mask"].sum(1)
    assert int(t5_len.min()) < 128 and int(t5_len.max()) == 128
    eos = g["tokenizers"]["clip_vocab"]["<|endoftext|>"]
    clip_len = (g["clip_ids"] != eos).sum(1) + 1
    assert int(clip_len.min()) < 77 and int(clip_len.max()) == 77
    assert g["flux"]["prompt_embeds"].abs().mean().item() > 0.1


def test_rebuilt_tokenizers_reproduce_the_stored_ids(golden_dir):
    g = torch.load(golden_dir / "text_encoder_small.pt", weights_only=False)
    tok = g["tokenizers"]
    clip = TO.clip_tokenizer(tok["clip_vocab"], tok["clip_merges"])
    t5 = TO.t5_tokenizer(tok["t5_tokenizer_json"])
    ids = clip(g["prompts"], padding="max_length", max_length=clip.model_max_length, truncation=True, return_tensors="pt")
    assert torch.equal(ids.input_ids, g["clip_ids"])
    t = t5(g["prompts"], padding="max_length", max_length=128, truncation=True, return_tensors="pt")
    assert torch.equal(t.input_ids, g["t5_ids"]) and torch.equal(t.attention_mask, g["t5_mask"])


@pytest.mark.parametrize("seq", [1, 7, 77, 128, 256])
def test_bias_table_matches_compute_bias(seq):
    from transformers.models.t5.modeling_t5 import T5Attention
    cfg = TO.hf_t5_config(TO.T5EncoderConfig(vocab_size=32, d_model=256, num_heads=4, num_layers=1, d_ff=512))
    att = T5Attention(cfg, has_relative_attention_bias=True)
    with torch.no_grad():
        att.relative_attention_bias.weight.copy_(torch.randn(32, 4, generator=torch.Generator().manual_seed(seq)))
        ref = att.compute_bias(seq, seq, device="cpu")[0]          # [heads, q, k]
    table = t5_bias_table(att.relative_attention_bias.weight, seq, 32, 128)
    assert table.shape == (4, 2 * seq - 1) and table.dtype == torch.float32
    q = torch.arange(seq)[:, None]
    k = torch.arange(seq)[None, :]
    assert torch.equal(table[:, k - q + seq - 1], ref)


def test_geglu_interleave_round_trip():
    g = torch.Generator().manual_seed(0)
    wi_0, wi_1 = torch.randn(320, 48, generator=g), torch.randn(320, 48, generator=g)
    w = interleave_geglu(wi_0, wi_1)
    assert w.shape == (640, 48)
    for t in range(5):   # tile t: gate rows [128 t, +64), linear rows [128 t + 64, +64)
        assert torch.equal(w[128 * t: 128 * t + 64], wi_0[64 * t: 64 * t + 64])
        assert torch.equal(w[128 * t + 64: 128 * t + 128], wi_1[64 * t: 64 * t + 64])
    a, b = deinterleave_geglu(w)
    assert torch.equal(a, wi_0) and torch.equal(b, wi_1)
    with pytest.raises(ValueError):
        interleave_geglu(torch.zeros(96, 8), torch.zeros(96, 8))


def test_clip_pooled_row_rules():
    ids = torch.tensor([[49406, 320, 49407, 0, 0], [49406, 49407, 5, 49407, 9]])
    # eos_token_id == 2: argmax of the ids (legacy); otherwise the first eos_token_id
    assert clip_pooled_index(ids, 2).tolist() == [2, 1]
    ids2 = torch.tensor([[1, 7, 5, 9, 5], [5, 5, 5, 5, 5]])
    assert clip_pooled_index(ids2, 5).tolist() == [2, 0]
    assert clip_pooled_index(ids2, 2).tolist() == [3, 0]
    for t, e in ((ids, 2), (ids, 49407), (ids2, 5), (ids2, 2)):
        assert torch.equal(clip_pooled_index(t, e), TO.clip_eos_index(t, e))


def _tiny_t5(**over):
    cfg = TO.T5EncoderConfig(vocab_size=32, d_model=128, num_heads=2, num_layers=1, d_ff=256)
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg, TO.synthetic_t5_params(TO.T5EncoderConfig(vocab_size=32, d_model=128, num_heads=2, num_layers=1, d_ff=256))


def _tiny_clip(**over):
    cfg = TO.ClipTextConfig(vocab_size=64, hidden_size=128, num_attention_heads=2, num_hidden_layers=1, intermediate_size=256)
    params = TO.synthetic_clip_params(cfg)
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg, params


def test_unsupported_configurations_raise():
    cfg, p = _tiny_t5(is_gated_act=False)
    with pytest.raises(ValueError, match="gated"):
        B200T5Encoder(cfg, p, device="cpu")
    cfg, p = _tiny_t5(dense_act_fn="relu")
    with pytest.raises(ValueError, match="dense_act_fn"):
        B200T5Encoder(cfg, p, device="cpu")
    cfg, p = _tiny_t5(d_kv=32)
    with pytest.raises(ValueError, match="head_dim"):
        B200T5Encoder(cfg, p, device="cpu")
    cfg, p = _tiny_clip(hidden_act="relu")
    with pytest.raises(ValueError, match="hidden_act"):
        B200CLIPText(cfg, p, device="cpu")
    cfg, p = _tiny_clip(num_attention_heads=4)
    with pytest.raises(ValueError, match="head_dim"):
        B200CLIPText(cfg, p, device="cpu")
    for act in ("quick_gelu", "gelu", "gelu_new", "gelu_pytorch_tanh"):
        cfg, p = _tiny_clip(hidden_act=act)
        B200CLIPText(cfg, p, device="cpu")


def test_bad_inputs_raise_before_any_launch():
    t5 = B200T5Encoder(*_tiny_t5(), device="cpu")
    ids = torch.randint(0, 32, (2, 16))
    mask = torch.ones(2, 16, dtype=torch.long)
    with pytest.raises(ValueError, match="out of range"):
        t5(torch.full((2, 16), 32), mask)
    with pytest.raises(ValueError, match="out of range"):
        t5(torch.full((2, 16), -1), mask)
    bad = mask.clone()
    bad[1] = 0
    with pytest.raises(ValueError, match="all zeros"):
        t5(ids, bad)
    clip = B200CLIPText(*_tiny_clip(), device="cpu")
    with pytest.raises(ValueError, match="out of range"):
        clip(torch.full((1, 77), 64))
    with pytest.raises(ValueError, match="max_position_embeddings"):
        clip(torch.zeros(1, 78, dtype=torch.long))
    # valid inputs with the weights on the CPU: no fallback
    with pytest.raises(RuntimeError, match="no CPU path"):
        t5(ids, mask)
    with pytest.raises(RuntimeError, match="no CPU path"):
        clip(torch.zeros(1, 77, dtype=torch.long))


def _err(lib):
    return lib.pf_last_error().decode()


def test_text_entry_points_validate_descriptors():
    lib = _lib.load()
    fake = 0x10000   # aligned, never dereferenced: every check below fails before a launch or a tensor map
    d = _lib.AttnTextDesc()
    assert lib.pf_attn_fwd_text(None, None) < 0
    assert lib.pf_attn_fwd_text(C.byref(d), None) < 0 and "null" in _err(lib)
    d.qkv, d.out, d.ld_qkv, d.ldo = fake, fake, 3 * 2 * 64, 2 * 64
    d.batch, d.heads, d.seq, d.head_dim, d.scale = 2, 2, 257, 64, 1.0
    assert lib.pf_attn_fwd_text(C.byref(d), None) < 0 and "exceeds 256" in _err(lib)
    d.seq, d.head_dim = 128, 128
    assert lib.pf_attn_fwd_text(C.byref(d), None) < 0 and "head_dim" in _err(lib)
    d.head_dim, d.ld_qkv = 64, 2 * 64
    assert lib.pf_attn_fwd_text(C.byref(d), None) < 0 and "ld_qkv" in _err(lib)

    assert lib.pf_rms_norm_rows(None, fake, fake, 1, 4, 0, 4, 128, 1e-6, None) < 0 and "null" in _err(lib)
    assert lib.pf_rms_norm_rows(fake, fake, fake, 1, 4, 2, 4, 128, 1e-6, None) < 0 and "row range" in _err(lib)
    assert lib.pf_embed_tokens(None, 4, 4, fake, 10, 128, None, 0, fake, None) < 0 and "null" in _err(lib)
    assert lib.pf_embed_tokens(fake, 8, 4, fake, 10, 128, fake, 3, fake, None) < 0 and "positions" in _err(lib)


def test_gemm_text_epilogues_validate():
    lib = _lib.load()
    fake = 0x10000
    d = _lib.GemmDesc()
    d.a, d.w, d.out = fake, fake, fake
    d.lda, d.k, d.batches, d.rows_per_batch, d.row_count = 64, 64, 1, 200, 200
    d.ldo, d.out_batch_rows = 64, 200
    d.n, d.epilogue = 192, _lib.PF_EPI_GEGLU_BF16
    assert lib.pf_gemm_bf16(C.byref(d), None) < 0 and "GEGLU needs n % 128 == 0" in _err(lib)
    d.n, d.kernel_variant = 256, 2
    assert lib.pf_gemm_bf16(C.byref(d), None) < 0 and "GEGLU" in _err(lib)
    d.kernel_variant, d.epilogue = 0, 17
    assert lib.pf_gemm_bf16(C.byref(d), None) < 0 and "unknown epilogue 17" in _err(lib)
    d.epilogue, d.lda, d.k = _lib.PF_EPI_QUICK_GELU_BF16, 128, 128
    assert lib.pf_gemm_fp8(C.byref(d), C.c_void_p(fake), C.c_void_p(fake), None) < 0 and "bf16 only" in _err(lib)
