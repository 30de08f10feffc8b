"""The FP8 (e4m3) GEMM path without a GPU: the host weight quantiser against the numerical contract of include/pf_b200.h,
host-side argument validation of the three fp8 entries, and which matrices the fp8 model imports as e4m3."""
import ctypes as C

import numpy as np
import pytest
import torch

from pyramid_flow_b200 import _lib, ops

E4M3_MAX = 448.0


def _contract_rows(w: torch.Tensor):
    """The contract restated row by row in numpy fp32 (IEEE division), the cast by torch."""
    x = w.float().numpy()
    q = np.empty_like(x)
    scale = np.empty(x.shape[0], np.float32)
    for r in range(x.shape[0]):
        amax = np.float32(np.abs(x[r]).max())
        inv = np.float32(E4M3_MAX) / amax if amax > 0 else np.float32(0)
        q[r] = x[r] * inv
        scale[r] = amax / np.float32(E4M3_MAX)
    return torch.from_numpy(q).to(torch.float8_e4m3fn), torch.from_numpy(scale)


def test_weight_quantiser_matches_the_contract():
    g = torch.Generator().manual_seed(3)
    w = torch.randn(64, 96, generator=g) * 0.02
    w[5] = 0.0                                            # zero row: zeros and scale 0
    w[6, :] = torch.randn(96, generator=g) * 3e30         # huge and tiny magnitudes: still finite
    w[7, :] = torch.randn(96, generator=g) * 1e-30
    w[8, 3] = -7.0                                        # the row's amax element maps to -448 exactly
    w8, s = ops.quantize_weight_fp8(w)
    q_ref, s_ref = _contract_rows(w)
    assert w8.dtype == torch.float8_e4m3fn and s.dtype == torch.float32 and w8.shape == w.shape and s.shape == (64,)
    assert torch.equal(w8.view(torch.uint8), q_ref.view(torch.uint8))
    assert torch.equal(s, s_ref)
    assert s[5].item() == 0.0 and bool((w8[5].float() == 0).all())
    assert bool(torch.isfinite(w8.float()).all()) and bool(torch.isfinite(s).all())
    assert w8[8, 3].float().item() == -E4M3_MAX
    assert w8.float().abs().max().item() <= E4M3_MAX
    # in the e4m3 normal range (|q| >= 2^-6) the dequantised value is within half an ulp (2^-4 relative) of the input
    deq = w8.float() * s[:, None]
    normal = w.abs() >= s[:, None] * 2.0 ** -6
    assert bool(((deq - w).abs() <= w.abs() * 2.0 ** -4)[normal].all())


def test_weight_quantiser_scale_is_an_ieee_division():
    """bf16-valued weights put many scaled values exactly on e4m3 rounding ties, where 448 * (1 / amax) (two roundings)
    and the contract's 448 / amax give different bits."""
    g = torch.Generator().manual_seed(5)
    w = (torch.randn(512, 64, generator=g) * torch.rand(512, 1, generator=g) * 5).bfloat16().float()
    w8, s = ops.quantize_weight_fp8(w)
    q_ref, s_ref = _contract_rows(w)
    assert torch.equal(w8.view(torch.uint8), q_ref.view(torch.uint8)) and torch.equal(s, s_ref)


def test_weight_quantiser_uses_the_fp32_values():
    """One rounding from the fp32 values: a bf16 detour would change some bits."""
    g = torch.Generator().manual_seed(4)
    w = torch.randn(32, 256, generator=g, dtype=torch.float64)
    w8, s = ops.quantize_weight_fp8(w)
    q_ref, s_ref = _contract_rows(w.float())
    assert torch.equal(w8.view(torch.uint8), q_ref.view(torch.uint8)) and torch.equal(s, s_ref)


def test_fp8_entries_reject_bad_arguments_with_a_message():
    """Validation is host-side and happens before any CUDA call.  Pointers are dummies, never dereferenced."""
    from pyramid_flow_b200._lib import PF_EPI_STORE_BF16, GemmDesc
    lib = _lib.load()
    dummy, scale = 0x1000, 0x2000

    def err():
        return lib.pf_last_error().decode()

    def desc():
        g = GemmDesc()
        g.a = g.w = g.out = dummy
        g.batches, g.rows_per_batch, g.row_count, g.n, g.k, g.lda, g.ldo = 1, 256, 256, 256, 128, 128, 256
        g.epilogue = PF_EPI_STORE_BF16
        return g

    assert lib.pf_gemm_fp8(None, scale, scale, None) < 0 and "null" in err()
    assert lib.pf_gemm_fp8(C.byref(desc()), None, scale, None) < 0 and "scale" in err()
    assert lib.pf_gemm_fp8(C.byref(desc()), scale, None, None) < 0 and "scale" in err()
    g = desc()
    g.peer_count = 2
    assert lib.pf_gemm_fp8(C.byref(g), scale, scale, None) < 0 and "peer" in err()
    g = desc()
    g.kernel_variant = 1
    assert lib.pf_gemm_fp8(C.byref(g), scale, scale, None) < 0 and "kernel_variant" in err()
    g = desc()
    g.n = 192
    assert lib.pf_gemm_fp8(C.byref(g), scale, scale, None) < 0 and "multiple of 128" in err()
    g = desc()
    g.k, g.lda = 120, 120
    assert lib.pf_gemm_fp8(C.byref(g), scale, scale, None) < 0 and "k=120" in err()
    g = desc()
    g.lda = 136
    assert lib.pf_gemm_fp8(C.byref(g), scale, scale, None) < 0 and "lda" in err()
    g = desc()
    g.epilogue = 17
    assert lib.pf_gemm_fp8(C.byref(g), scale, scale, None) < 0 and "epilogue" in err()

    assert lib.pf_ln_modulate_fp8(dummy, dummy, None, 1, 8, 0, 8, 256, dummy, dummy, 512, 1e-6, None) < 0 and "null" in err()
    assert lib.pf_ln_modulate_fp8(dummy, dummy, scale, 1, 8, 0, 8, 200, dummy, dummy, 512, 1e-6, None) < 0 and "dim" in err()
    assert lib.pf_ln_modulate_fp8(dummy, dummy, scale, 1, 8, 4, 8, 256, dummy, dummy, 512, 1e-6, None) < 0 and "row" in err()

    assert lib.pf_quantize_rows_fp8(dummy, 256, dummy, 256, None, 1, 8, 0, 8, 256, None) < 0 and "null" in err()
    assert lib.pf_quantize_rows_fp8(dummy, 256, dummy, 256, scale, 1, 8, 0, 8, 100, None) < 0 and "cols" in err()
    assert lib.pf_quantize_rows_fp8(dummy, 252, dummy, 256, scale, 1, 8, 0, 8, 248, None) < 0 and "ldx" in err()
    assert lib.pf_quantize_rows_fp8(dummy, 256, dummy, 128, scale, 1, 8, 0, 8, 256, None) < 0 and "ldy" in err()
    assert lib.pf_quantize_rows_fp8(dummy + 8, 256, dummy, 256, scale, 1, 8, 0, 8, 256, None) < 0 and "aligned" in err()
    assert lib.pf_quantize_rows_fp8(dummy, 256, dummy, 256, scale, 2, 8, 6, 4, 256, None) < 0 and "row range" in err()


def _tiny_fp8_model(precision):
    from oracle import flux_oracle as FO
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    kw = dict(num_layers=2, num_single_layers=2, num_attention_heads=4, attention_head_dim=64, in_channels=64,
              joint_attention_dim=128, pooled_projection_dim=64)
    params = FO.synthetic_flux_params(FO.FluxConfig(**kw), seed=0)
    return B200FluxTransformer(FluxConfigB200(**kw), params, device="cpu", gemm_precision=precision), params


FP8_DOUBLE = {"w_qkv": (".attn.to_q", ".attn.to_k", ".attn.to_v"), "w_o": (".attn.to_out.0",), "w_f1": (".ff.net.0.proj",),
              "w_f2": (".ff.net.2",)}
FP8_SINGLE = {"w_qkv": (".attn.to_q", ".attn.to_k", ".attn.to_v"), "w_mlp": (".proj_mlp",), "w_out": (".proj_out",)}


def test_fp8_model_imports_e4m3_weights_for_exactly_the_listed_gemms():
    model, params = _tiny_fp8_model("fp8")
    expected = set()
    for i, blk in enumerate(model.dbl):
        for key, parts in FP8_DOUBLE.items():
            expected.add(f"dbl{i}_{key}")
            w8, s = blk[key], blk["s" + key[1:]]
            want_w8, want_s = ops.quantize_weight_fp8(torch.cat([params[f"transformer_blocks.{i}{p}.weight"] for p in parts]))
            assert torch.equal(w8.view(torch.uint8), want_w8.view(torch.uint8)) and torch.equal(s, want_s)
        for key in ("w_cqkv", "w_co", "w_cf1", "w_cf2"):                      # text stream stays bf16
            assert blk[key].dtype == torch.bfloat16
    for i, blk in enumerate(model.sgl):
        for key, parts in FP8_SINGLE.items():
            expected.add(f"sgl{i}_{key}")
            want_w8, want_s = ops.quantize_weight_fp8(
                torch.cat([params[f"single_transformer_blocks.{i}{p}.weight"] for p in parts]))
            assert torch.equal(blk[key].view(torch.uint8), want_w8.view(torch.uint8))
            assert torch.equal(blk["s" + key[1:]], want_s)
    bufs = dict(model.named_buffers())
    fp8 = {n for n, t in bufs.items() if t.dtype == torch.float8_e4m3fn}
    assert fp8 == expected
    for n in expected:                                                    # fp32 scale per output channel, no bf16 copy
        sc = bufs[n.replace("_w_", "_s_")]
        assert sc.dtype == torch.float32 and sc.shape == (bufs[n].shape[0],)
    for n in ("w_x", "w_ctx", "w_out", "w_mod", "w_t1", "w_p1"):            # embedders, head, conditioning stay bf16
        assert bufs[n].dtype == torch.bfloat16
    bf16_model, _ = _tiny_fp8_model("bf16")
    assert not any(t.dtype == torch.float8_e4m3fn for t in bf16_model.buffers())
    assert {n for n in dict(bf16_model.named_buffers())} == {n for n in bufs if "_s_" not in n}


def test_fp8_model_rejects_unknown_precision_and_parallel_layouts():
    from oracle import flux_oracle as FO
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    with pytest.raises(ValueError, match="gemm_precision"):
        B200FluxTransformer(FluxConfigB200(num_layers=1, num_single_layers=1),
                            FO.synthetic_flux_params(FO.FluxConfig(num_layers=1, num_single_layers=1), seed=0),
                            device="cpu", gemm_precision="fp16")
    model, _ = _tiny_fp8_model("fp8")
    with pytest.raises(NotImplementedError, match="fp8"):
        model.set_parallel_layout(object())
