"""The SD3 MMDiT's gemm_precision="fp8" without a GPU: which matrices it imports as e4m3 (the video stream's QKV, to_out, FF1
and FF2 of every joint block), their bits and scales, what stays bf16, and the rejected configurations."""
import pytest
import torch

from pyramid_flow_b200 import ops

FP8_BLOCK = {"w_qkv": (".attn.to_q", ".attn.to_k", ".attn.to_v"), "w_o": (".attn.to_out.0",), "w_f1": (".ff.net.0.proj",),
             "w_f2": (".ff.net.2",)}
TEXT_BLOCK = ("w_cqkv", "w_co", "w_cf1", "w_cf2")


def _tiny_mmdit(precision=None, num_layers=3):
    from oracle import mmdit_oracle as MO
    from pyramid_flow_b200.mmdit import B200MMDiT, MMDiTConfigB200
    kw = dict(num_layers=num_layers, num_attention_heads=4, attention_head_dim=64, in_channels=16, joint_attention_dim=128,
              pooled_projection_dim=64, pos_embed_max_size=16)
    params = MO.synthetic_mmdit_params(MO.MMDiTConfig(sample_size=16, **kw), seed=0)
    prec = {} if precision is None else dict(gemm_precision=precision)
    return B200MMDiT(MMDiTConfigB200(**kw), params, device="cpu", **prec), params


def test_fp8_mmdit_imports_e4m3_weights_for_exactly_the_video_block_gemms():
    model, params = _tiny_mmdit("fp8")
    expected = set()
    for i, blk in enumerate(model.blocks):
        last = i == len(model.blocks) - 1
        for key, parts in FP8_BLOCK.items():         # the context_pre_only last block's video stream included
            expected.add(f"blk{i}_{key}")
            want_w8, want_s = ops.quantize_weight_fp8(torch.cat([params[f"transformer_blocks.{i}{p}.weight"] for p in parts]))
            assert torch.equal(blk[key].view(torch.uint8), want_w8.view(torch.uint8))
            assert torch.equal(blk["s" + key[1:]], want_s)
        for key in TEXT_BLOCK[:1] if last else TEXT_BLOCK:                   # text stream stays bf16
            assert blk[key].dtype == torch.bfloat16
        assert last == ("w_co" not in blk)
    bufs = dict(model.named_buffers())
    assert {n for n, t in bufs.items() if t.dtype == torch.float8_e4m3fn} == expected
    for n in expected:                                                    # fp32 scale per output channel, no bf16 copy
        sc = bufs[n.replace("_w_", "_s_")]
        assert sc.dtype == torch.float32 and sc.shape == (bufs[n].shape[0],)
    for n in ("w_x", "w_ctx", "w_out", "w_mod", "w_t1", "w_t2", "w_p1", "w_p2"):   # embedders, head, conditioning stay bf16
        assert bufs[n].dtype == torch.bfloat16
    bf16_model, _ = _tiny_mmdit("bf16")
    assert not any(t.dtype == torch.float8_e4m3fn for t in bf16_model.buffers())
    assert set(dict(bf16_model.named_buffers())) == {n for n in bufs if "_s_" not in n}


def test_default_precision_is_bf16_with_the_same_weights():
    model, _ = _tiny_mmdit("bf16")
    default, _ = _tiny_mmdit()
    assert default.gemm_precision == "bf16"
    a, b = dict(model.named_buffers()), dict(default.named_buffers())
    assert set(a) == set(b) and all(torch.equal(a[n], b[n]) for n in a)


def test_fp8_mmdit_rejects_unknown_precision_and_parallel_layouts():
    with pytest.raises(ValueError, match="gemm_precision"):
        _tiny_mmdit("fp16", num_layers=1)
    model, _ = _tiny_mmdit("fp8", num_layers=1)
    with pytest.raises(NotImplementedError, match="fp8"):
        model.set_parallel_layout(object())


def test_from_reference_passes_the_precision():
    from types import SimpleNamespace
    from pyramid_flow_b200.mmdit import B200MMDiT
    model, params = _tiny_mmdit("fp8", num_layers=1)
    c = model.cfg
    ref = SimpleNamespace(config=SimpleNamespace(num_layers=c.num_layers, num_attention_heads=c.num_attention_heads,
                                                 attention_head_dim=c.attention_head_dim, in_channels=c.in_channels,
                                                 patch_size=c.patch_size, joint_attention_dim=c.joint_attention_dim,
                                                 pooled_projection_dim=c.pooled_projection_dim,
                                                 pos_embed_max_size=c.pos_embed_max_size),
                          state_dict=lambda: params)
    m8 = B200MMDiT.from_reference(ref, device="cpu", gemm_precision="fp8")
    assert m8.gemm_precision == "fp8" and m8.blocks[0]["w_f1"].dtype == torch.float8_e4m3fn
    assert B200MMDiT.from_reference(ref, device="cpu").blocks[0]["w_f1"].dtype == torch.bfloat16
    with pytest.raises(ValueError, match="gemm_precision"):
        B200MMDiT.from_reference(ref, device="cpu", gemm_precision="int8")
