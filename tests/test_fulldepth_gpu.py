"""Parity at FULL DEPTH and full size: the model the bench times (8 double + 16 single miniFLUX blocks, D=1920, 30 heads, B=2,
S=15488 = 768p unit 30 / stage 2) against the fp32 oracle evaluated on the same GPU (TF32 off, math SDPA a few heads at a
time), plus the 24-block SD3 MMDiT.  Reports the error at depth next to the shallow-model figure of tests/test_dit_gpu.py so
that error growth over the 24 blocks is visible, and an fp32-output figure that separates the bf16 store of the velocity from
the operand error.

Stated tolerance (per-step velocity vs the fp32 oracle on identical inputs, |v| ~ 0.9): see TOL_* below = measured x 1.3."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# Thresholds = 1.3 x the error of the first implementation of these kernels; the sm_90a kernels are held to the same ones.
TOL_FULL_MAX_ABS = 1.5e-2       # fp32 velocity store
TOL_FULL_MSE = 7.6e-6
TOL_FULL_BF16_MAX_ABS = 2.5e-2  # bf16 velocity store (what the pipeline receives): |v| reaches 5.6 here, where
TOL_FULL_BF16_MSE = 1.22e-5     # half a bf16 ulp is 1.6e-2
TOL_MMDIT24_MAX_ABS = 1.47e-2
TOL_MMDIT24_MSE = 8.0e-6


def _oracle_on_gpu(fn, head_chunk):
    from oracle import flux_oracle as FO
    from torch.nn.attention import SDPBackend, sdpa_kernel
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    FO.HEAD_CHUNK = head_chunk
    try:
        with torch.no_grad(), sdpa_kernel(SDPBackend.MATH):
            return fn()
    finally:
        FO.HEAD_CHUNK = 0


def test_full_depth_full_size_flux_step_matches_oracle():
    from oracle import flux_oracle as FO
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    dev = torch.device("cuda:0")
    cfg = FO.FluxConfig()                                   # 8 + 16 blocks, D=1920, 30 heads
    params = FO.synthetic_flux_params(cfg, seed=11)
    gen = torch.Generator().manual_seed(12)
    shapes = [(2, 16, 28, 24, 40), (2, 16, 1, 48, 80), (2, 16, 1, 96, 160), (2, 16, 1, 96, 160)]
    clips = [torch.randn(s, generator=gen).bfloat16().float() for s in shapes]
    enc = (torch.randn(2, 128, 4096, generator=gen) * 0.2).bfloat16().float()
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[0, 77:] = 0
    pooled = torch.randn(2, 768, generator=gen)
    t = torch.tensor([3.0, 3.0])

    model = B200FluxTransformer(FluxConfigB200(), params, device=dev)
    call = dict(sample=[[c.to(dev).bfloat16() for c in clips]], timestep_ratio=t.to(dev), encoder_hidden_states=enc.to(dev),
                encoder_attention_mask=mask.to(dev), pooled_projections=pooled.to(dev))
    o = model(**call)[0]                                  # bf16 latents in -> bf16 velocity out (what the pipeline sees)
    assert o.dtype == torch.bfloat16 and model.last_plan.seq == 15488
    out = o.float().cpu()
    model.output_fp32 = True                              # same step, velocity stored in fp32: isolates the bf16 store
    o32 = model(**call)[0]
    assert o32.dtype == torch.float32
    out32 = o32.float().cpu()
    model.output_fp32 = False

    pd = {k: v.to(dev) for k, v in params.items()}
    del params
    ref = _oracle_on_gpu(lambda: FO.flux_forward(pd, cfg, [c.to(dev) for c in clips], t.to(dev), enc.to(dev), mask,
                                                 pooled.to(dev)).float().cpu(), head_chunk=3)
    del pd
    torch.cuda.empty_cache()
    err, mse = (out - ref).abs().max().item(), ((out - ref) ** 2).mean().item()
    err32, mse32 = (out32 - ref).abs().max().item(), ((out32 - ref) ** 2).mean().item()
    print(f"FULL DEPTH 8+16 @ S=15488: bf16-out max_abs {err:.3e} mse {mse:.3e} | fp32-out max_abs {err32:.3e} mse {mse32:.3e} "
          f"| |v| mean {ref.abs().mean():.3f} max {ref.abs().max():.2f}")
    assert ref.abs().mean().item() > 0.1, "degenerate oracle output"
    assert err32 < TOL_FULL_MAX_ABS and mse32 < TOL_FULL_MSE
    assert err < TOL_FULL_BF16_MAX_ABS and mse < TOL_FULL_BF16_MSE
    assert mse32 <= mse      # the bf16 store can only add error


def test_24_block_mmdit_step_matches_oracle():
    """SD3 MMDiT at its real depth (24 joint blocks incl. the context-pre-only last one, D=1536, 24 heads), 384p-like pyramid
    with ragged text (S = 128 + 1320)."""
    from oracle import mmdit_oracle as MO
    from pyramid_flow_b200.mmdit import B200MMDiT, MMDiTConfigB200
    dev = torch.device("cuda:0")
    kw = dict(num_layers=24, pos_embed_max_size=96, sample_size=64)
    cfg = MO.MMDiTConfig(**kw)
    params = MO.synthetic_mmdit_params(cfg, seed=21)
    g = torch.Generator().manual_seed(22)
    clips = [torch.randn(2, 16, 2, 12, 20, generator=g), torch.randn(2, 16, 1, 24, 40, generator=g),
             torch.randn(2, 16, 1, 48, 80, generator=g)]
    clips = [c.bfloat16().float() for c in clips]
    enc = (torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().float()
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[1, 61:] = 0
    pooled = torch.randn(2, 2048, generator=g)
    t = torch.tensor([640.0, 640.0])
    mkw = {k: v for k, v in kw.items() if k != "sample_size"}
    model = B200MMDiT(MMDiTConfigB200(**mkw), params, device=dev)
    out = model(sample=[[c.to(dev) for c in clips]], timestep_ratio=t.to(dev), encoder_hidden_states=enc.to(dev),
                encoder_attention_mask=mask.to(dev), pooled_projections=pooled.to(dev))[0].float().cpu()
    pd = {k: v.to(dev) for k, v in params.items()}
    ref = _oracle_on_gpu(lambda: MO.mmdit_forward(pd, cfg, [c.to(dev) for c in clips], t.to(dev), enc.to(dev), mask,
                                                  pooled.to(dev)).float().cpu(), head_chunk=0)
    err, mse = (out - ref).abs().max().item(), ((out - ref) ** 2).mean().item()
    print(f"MMDiT 24 blocks: max_abs {err:.3e} mse {mse:.3e} | |v| mean {ref.abs().mean():.3f}")
    assert ref.abs().mean().item() > 0.1
    assert err < TOL_MMDIT24_MAX_ABS and mse < TOL_MMDIT24_MSE
