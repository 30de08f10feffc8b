"""Generate tests/golden/text_encoder_small.pt: what the UNMODIFIED reference text-encoder wrappers compute, pinning
oracle/text_encoder_oracle.py.

    python oracle/pin/make_text_golden.py      (CPU, fp32; needs a readable reference checkout, see oracle/pin/ref_shim.py)

FluxTextEncoderWithMask (pyramid_dit/flux_modules/modeling_text_encoder.py) and SD3TextEncoderWithMask
(pyramid_dit/mmdit_modules/modeling_text_encoder.py) are built by __new__ with tiny transformers models (CLIPTextModel /
CLIPTextModelWithProjection / T5EncoderModel) holding the oracle's synthetic parameters, loaded with strict=True, and tiny
tokenizers: a byte-level BPE CLIPTokenizer and a word-level `tokenizers` model in a T5TokenizerFast.  Their definitions,
the prompts, the token ids / masks and the three outputs of forward(prompts, "cpu") are stored.  The prompts cover padded
and unpadded sequences (an unpadded CLIP prompt, an unpadded T5 prompt) and truncation (both tokenizers).  Flux's CLIP and
SD3's CLIP-L take the legacy pooled-row rule (eos_token_id = 2), SD3's CLIP-G the first-EOS rule.  Both wrappers hold the
same T5 (same configuration and seed), so their T5 outputs must be equal; the script checks that and stores the tensor
once (both entries refer to it), which keeps the fixture small.
"""
from __future__ import annotations

import sys
from dataclasses import asdict
from pathlib import Path

import torch
import torch.nn as nn

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle.pin import ref_shim  # noqa: E402

ref_shim.install()
from oracle import text_encoder_oracle as TO  # noqa: E402

GOLD = ROOT / "tests" / "golden"

T5_WORDS = "a cat dog sat on the mat photo of red blue green small big house tree in under over river sky".split()
CLIP_MERGES = ["a t</w>", "c a", "ca t</w>", "d o", "do g</w>", "r e", "re d</w>", "t h", "th e</w>"]
PROMPTS = [
    "a red cat",                                 # padded by both
    "a " * 75,                                   # 77 CLIP tokens with BOS / EOS: unpadded for CLIP
    "photo " * 127,                              # 128 T5 tokens with EOS: unpadded for T5, truncated for CLIP
    "a big green tree under the blue sky " * 30,  # truncated by both
]
SEEDS = dict(flux_clip=11, flux_t5=12, sd3_clip_l=13, sd3_clip_g=14, sd3_t5=12)   # one T5 for both wrappers


def tokenizer_definitions():
    from tokenizers import Tokenizer, models, pre_tokenizers, processors
    from tokenizers.pre_tokenizers import ByteLevel
    chars = sorted(ByteLevel.alphabet())
    vocab = {c: i for i, c in enumerate(chars)}
    for c in chars:
        vocab[c + "</w>"] = len(vocab)
    for m in CLIP_MERGES:
        a, b = m.split()
        vocab[a + b] = len(vocab)
    vocab["<|startoftext|>"] = len(vocab)
    vocab["<|endoftext|>"] = len(vocab)
    words = {"<pad>": 0, "</s>": 1, "<unk>": 2}
    for w in T5_WORDS:
        words["▁" + w] = len(words)
    t5 = Tokenizer(models.WordLevel(words, unk_token="<unk>"))
    t5.pre_tokenizer = pre_tokenizers.Metaspace()
    t5.post_processor = processors.TemplateProcessing(single="$A </s>", special_tokens=[("</s>", 1)])
    return {"clip_vocab": vocab, "clip_merges": CLIP_MERGES, "t5_tokenizer_json": t5.to_str()}


def configs(tok):
    clip_vocab = len(tok["clip_vocab"])
    eos = tok["clip_vocab"]["<|endoftext|>"]
    clip = dict(vocab_size=clip_vocab, hidden_size=128, num_attention_heads=2, num_hidden_layers=2, intermediate_size=256)
    t5 = TO.T5EncoderConfig(vocab_size=32, d_model=128, num_heads=2, num_layers=2, d_ff=256)
    return {
        "flux_clip": TO.ClipTextConfig(**clip, hidden_act="quick_gelu", eos_token_id=2),
        "flux_t5": t5,
        "sd3_clip_l": TO.ClipTextConfig(**clip, hidden_act="quick_gelu", eos_token_id=2, projection_dim=128),
        "sd3_clip_g": TO.ClipTextConfig(vocab_size=clip_vocab, hidden_size=256, num_attention_heads=4, num_hidden_layers=2,
                                        intermediate_size=512, hidden_act="gelu", eos_token_id=eos, projection_dim=128),
        "sd3_t5": t5,
    }


def build_wrappers(tok, cfgs, params):
    """The unmodified reference wrappers around tiny transformers models; params[name] are the oracle's parameters."""
    from pyramid_dit.flux_modules.modeling_text_encoder import FluxTextEncoderWithMask
    from pyramid_dit.mmdit_modules.modeling_text_encoder import SD3TextEncoderWithMask

    def clip_tok():
        return TO.clip_tokenizer(tok["clip_vocab"], tok["clip_merges"])

    flux = FluxTextEncoderWithMask.__new__(FluxTextEncoderWithMask)
    nn.Module.__init__(flux)
    flux.tokenizer = clip_tok()
    flux.tokenizer_max_length = flux.tokenizer.model_max_length
    flux.text_encoder = TO.hf_clip_model(cfgs["flux_clip"], params["flux_clip"])
    flux.tokenizer_2 = TO.t5_tokenizer(tok["t5_tokenizer_json"])
    flux.text_encoder_2 = TO.hf_t5_model(cfgs["flux_t5"], params["flux_t5"])
    flux._freeze()

    sd3 = SD3TextEncoderWithMask.__new__(SD3TextEncoderWithMask)
    nn.Module.__init__(sd3)
    sd3.tokenizer = clip_tok()
    sd3.tokenizer_max_length = sd3.tokenizer.model_max_length
    sd3.text_encoder = TO.hf_clip_model(cfgs["sd3_clip_l"], params["sd3_clip_l"])
    sd3.tokenizer_2 = clip_tok()
    sd3.text_encoder_2 = TO.hf_clip_model(cfgs["sd3_clip_g"], params["sd3_clip_g"])
    sd3.tokenizer_3 = TO.t5_tokenizer(tok["t5_tokenizer_json"])
    sd3.text_encoder_3 = TO.hf_t5_model(cfgs["sd3_t5"], params["sd3_t5"])
    sd3._freeze()
    return flux, sd3


def synthetic_params(cfgs):
    return {name: (TO.synthetic_clip_params if isinstance(cfg, TO.ClipTextConfig) else TO.synthetic_t5_params)(cfg, SEEDS[name])
            for name, cfg in cfgs.items()}


def main() -> None:
    tok = tokenizer_definitions()
    cfgs = configs(tok)
    params = synthetic_params(cfgs)
    flux, sd3 = build_wrappers(tok, cfgs, params)
    out = {"tokenizers": tok, "configs": {k: asdict(v) for k, v in cfgs.items()}, "seeds": SEEDS, "prompts": PROMPTS}
    clip_in = flux.tokenizer(PROMPTS, padding="max_length", max_length=flux.tokenizer_max_length, truncation=True,
                             return_tensors="pt")
    t5_in = flux.tokenizer_2(PROMPTS, padding="max_length", max_length=128, truncation=True, return_tensors="pt")
    out["clip_ids"] = clip_in.input_ids
    out["t5_ids"], out["t5_mask"] = t5_in.input_ids, t5_in.attention_mask
    with torch.no_grad():
        for name, w in (("flux", flux), ("sd3", sd3)):
            pe, am, pooled = w(PROMPTS, "cpu")
            if name == "sd3":      # the same T5: the tensors are stored once
                assert torch.equal(pe, out["flux"]["prompt_embeds"]) and torch.equal(am, out["flux"]["prompt_attention_mask"])
                pe, am = out["flux"]["prompt_embeds"], out["flux"]["prompt_attention_mask"]
            out[name] = {"prompt_embeds": pe, "prompt_attention_mask": am, "pooled_prompt_embeds": pooled}
            print(f"[make_text_golden] {name}: {tuple(pe.shape)} {pe.dtype} {tuple(am.shape)} {am.dtype} {tuple(pooled.shape)} "
                  f"|embeds| {float(pe.abs().mean()):.4f} |pooled| {float(pooled.abs().mean()):.4f}")
    print("[make_text_golden] T5 tokens per prompt", out["t5_mask"].sum(1).tolist(), "CLIP EOS positions",
          TO.clip_eos_index(out["clip_ids"], 2).tolist())
    torch.save(out, GOLD / "text_encoder_small.pt")


if __name__ == "__main__":
    main()
