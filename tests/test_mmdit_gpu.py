"""Parity of the CUDA SD3-MMDiT step (BASELINE configs[4] path) against the reference golden / oracle. Needs an H100."""
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL_MAX_ABS = 1.55e-2
TOL_MSE = 6e-6


def _run(cfg_kw, params, clips, t, enc, mask, pooled):
    from pyramid_flow_b200.mmdit import B200MMDiT, MMDiTConfigB200
    dev = torch.device("cuda:0")
    kw = {k: v for k, v in cfg_kw.items() if k != "sample_size"}
    model = B200MMDiT(MMDiTConfigB200(**kw), params, device=dev)
    out = model(sample=[[c.to(dev) for c in clips]], timestep_ratio=t.to(dev), encoder_hidden_states=enc.to(dev),
                encoder_attention_mask=mask.to(dev), pooled_projections=pooled.to(dev))[0]
    torch.cuda.synchronize()
    return out.float().cpu()


def test_small_mmdit_matches_reference_golden(golden_dir):
    from oracle import mmdit_oracle as MO
    g = torch.load(golden_dir / "mmdit_small.pt", weights_only=False)
    cfg = MO.MMDiTConfig(**g["cfg"])
    params = MO.synthetic_mmdit_params(cfg, seed=g["param_seed"])
    enc = g["enc"].bfloat16().float()
    clips = [c.bfloat16().float() for c in g["clips"]]
    with torch.no_grad():
        ref = MO.mmdit_forward(params, cfg, clips, g["timestep"], enc, g["mask"], g["pooled"])
    out = _run(g["cfg"], params, clips, g["timestep"], enc, g["mask"], g["pooled"])
    err, mse = (out - ref).abs().max().item(), ((out - ref) ** 2).mean().item()
    err_gold = (out - g["out"]).abs().max().item()
    print(f"mmdit small: max_abs vs oracle {err:.3e} mse {mse:.3e}; vs reference golden {err_gold:.3e}")
    assert err < TOL_MAX_ABS and mse < TOL_MSE and err_gold < TOL_MAX_ABS


def test_sd3_width_mmdit_matches_oracle():
    """SD3 width (D=1536, 24 heads), 3 blocks (incl. the context_pre_only last block), 384p-like pyramid."""
    from oracle import mmdit_oracle as MO
    kw = dict(num_layers=3, pos_embed_max_size=96, sample_size=64)
    cfg = MO.MMDiTConfig(**kw)
    params = MO.synthetic_mmdit_params(cfg, seed=2)
    g = torch.Generator().manual_seed(6)
    clips = [torch.randn(2, 16, 2, 12, 20, generator=g), torch.randn(2, 16, 1, 24, 40, generator=g),
             torch.randn(2, 16, 1, 48, 80, generator=g)]
    clips = [c.bfloat16().float() for c in clips]
    enc = (torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().float()
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[0, 50:] = 0
    pooled = torch.randn(2, 2048, generator=g)
    t = torch.tensor([500.0, 500.0])
    dev = torch.device("cuda:0")
    pd = {k: v.to(dev) for k, v in params.items()}
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from torch.nn.attention import SDPBackend, sdpa_kernel
    with torch.no_grad(), sdpa_kernel(SDPBackend.MATH):
        ref = MO.mmdit_forward(pd, cfg, [c.to(dev) for c in clips], t.to(dev), enc.to(dev), mask, pooled.to(dev)).float().cpu()
    out = _run(kw, params, clips, t, enc, mask, pooled)
    err, mse = (out - ref).abs().max().item(), ((out - ref) ** 2).mean().item()
    print(f"mmdit sd3-width: max_abs {err:.3e} mse {mse:.3e} |v| mean {ref.abs().mean():.3f}")
    assert err < TOL_MAX_ABS and mse < TOL_MSE
