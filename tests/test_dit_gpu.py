"""Parity of the CUDA DiT step (through the C-ABI) against the oracle / the reference's golden outputs. Needs an H100."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# Stated tolerance (BASELINE.json north_star: per-step velocity max-abs vs the reference on identical inputs).
# Velocities are O(1) (|v| mean ~0.9 for the synthetic weights); all GEMM/attention operands are bf16 (ulp(1) = 7.8e-3),
# accumulation, LN/RMS statistics, softmax and the residual stream are fp32.  Measured error is reported next to the
# error of the reference's own dtype policy (oracle under bf16 autocast) against the same fp32 truth.
# Thresholds = 1.3 x the error of the first implementation of these kernels; the sm_90a kernels are held to the same ones.
TOL_MAX_ABS = 1.5e-2
TOL_MSE = 6e-6


def _to(dev, *xs):
    return [x.to(dev) for x in xs]


def _run_ours(kw, params, clips, t, enc, mask, pooled):
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    dev = torch.device("cuda:0")
    model = B200FluxTransformer(FluxConfigB200(**kw), params, device=dev)
    out = model(sample=[[c.to(dev) for c in clips]], timestep_ratio=t.to(dev), encoder_hidden_states=enc.to(dev),
                encoder_attention_mask=mask.to(dev), pooled_projections=pooled.to(dev))[0]
    torch.cuda.synchronize()
    return out.float().cpu(), model


def test_small_step_matches_reference_golden(golden_dir):
    from oracle import flux_oracle as FO
    g = torch.load(golden_dir / "flux_small.pt", weights_only=False)
    cfg = FO.FluxConfig(**g["cfg"])
    params = FO.synthetic_flux_params(cfg, seed=g["param_seed"])
    # the CUDA path consumes bf16 latents / text embeddings (what the pipeline provides): round once, feed both sides
    enc = g["enc"].bfloat16().float()
    clips = [c.bfloat16().float() for c in g["clips"]]
    with torch.no_grad():
        ref = FO.flux_forward(params, cfg, clips, g["timestep"], enc, g["mask"], g["pooled"])
    out, _ = _run_ours(g["cfg"], params, clips, g["timestep"], enc, g["mask"], g["pooled"])
    err = (out - ref).abs().max().item()
    err_gold = (out - g["out"]).abs().max().item()   # vs the unmodified reference's fp32 output (enc not rounded)
    mse = ((out - ref) ** 2).mean().item()
    print(f"small: max_abs vs oracle {err:.3e}, vs reference golden {err_gold:.3e}, mse {mse:.3e}")
    assert err < TOL_MAX_ABS and err_gold < TOL_MAX_ABS and mse < TOL_MSE
    # first-unit shape (single clip) and full mask
    out1, _ = _run_ours(g["cfg"], params, [g["clips"][-1]], g["timestep"] * 0.5, enc, g["mask"], g["pooled"])
    assert (out1 - g["out_first"]).abs().max().item() < TOL_MAX_ABS
    out2, _ = _run_ours(g["cfg"], params, g["clips"], g["timestep"], enc, torch.ones_like(g["mask"]), g["pooled"])
    assert (out2 - g["out_full_mask"]).abs().max().item() < TOL_MAX_ABS


def test_miniflux_width_step_matches_oracle():
    """miniFLUX width (D=1920, 30 heads), 2+2 blocks, 384p-like pyramid (S=1448), B=2 with ragged text."""
    from oracle import flux_oracle as FO
    kw = dict(num_layers=2, num_single_layers=2)
    cfg = FO.FluxConfig(**kw)
    dev = torch.device("cuda:0")
    params = FO.synthetic_flux_params(cfg, seed=3)
    g = torch.Generator().manual_seed(4)
    clips = [torch.randn(2, 16, 2, 12, 20, generator=g), torch.randn(2, 16, 1, 24, 40, generator=g),
             torch.randn(2, 16, 1, 48, 80, generator=g)]
    clips = [c.bfloat16().float() for c in clips]
    enc = (torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().float()
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[0, 37:] = 0
    pooled = torch.randn(2, 768, generator=g)
    t = torch.tensor([744.0, 744.0])
    pd = {k: v.to(dev) for k, v in params.items()}
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from torch.nn.attention import SDPBackend, sdpa_kernel
    with torch.no_grad(), sdpa_kernel(SDPBackend.MATH):
        ref = FO.flux_forward(pd, cfg, _to(dev, *clips), t.to(dev), enc.to(dev), mask, pooled.to(dev)).float().cpu()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ref_bf16 = FO.flux_forward(pd, cfg, [c.to(dev).bfloat16() for c in clips], t.to(dev).bfloat16(),
                                       enc.to(dev).bfloat16(), mask, pooled.to(dev).bfloat16()).float().cpu()
    out, model = _run_ours(kw, params, clips, t, enc, mask, pooled)
    err = (out - ref).abs().max().item()
    mse = ((out - ref) ** 2).mean().item()
    err_ref_bf16 = (ref_bf16 - ref).abs().max().item()
    mse_ref_bf16 = ((ref_bf16 - ref) ** 2).mean().item()
    print(f"miniflux-width: ours vs fp32 oracle max_abs {err:.3e} mse {mse:.3e} | reference dtype policy (bf16 autocast) "
          f"vs fp32 oracle max_abs {err_ref_bf16:.3e} mse {mse_ref_bf16:.3e} | |v| mean {ref.abs().mean():.3f}")
    assert err < TOL_MAX_ABS and mse < TOL_MSE
    assert err <= 1.5 * err_ref_bf16 + 2e-3, "CUDA path must be at least as close to fp32 truth as the reference's bf16 path"
    # sample 1 (full text) must not depend on sample 0's padding pattern; and the output must be non-degenerate
    assert ref.abs().mean().item() > 0.1


def test_cuda_graph_replay_equals_host_launched_step(golden_dir):
    """The captured-graph path (use_cuda_graph) replays the same kernels: outputs are bit-identical to the host-launched
    step, for the capture call, for replays with new inputs, and after switching shapes and back."""
    from oracle import flux_oracle as FO
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    g = torch.load(golden_dir / "flux_small.pt", weights_only=False)
    cfg = FO.FluxConfig(**g["cfg"])
    params = FO.synthetic_flux_params(cfg, seed=g["param_seed"])
    dev = torch.device("cuda:0")
    model = B200FluxTransformer(FluxConfigB200(**g["cfg"]), params, device=dev)
    enc, mask, pooled = g["enc"].bfloat16().to(dev), g["mask"].to(dev), g["pooled"].to(dev)

    def call(clips, t):
        return model(sample=[[c.to(dev) for c in clips]], timestep_ratio=t.to(dev), encoder_hidden_states=enc,
                     encoder_attention_mask=mask, pooled_projections=pooled)[0].float().cpu()

    gen = torch.Generator().manual_seed(9)
    variants = [([c.bfloat16() for c in g["clips"]], g["timestep"]),
                ([torch.randn(c.shape, generator=gen).bfloat16() for c in g["clips"]], g["timestep"] * 0.25),
                ([g["clips"][-1].bfloat16()], g["timestep"] * 0.5)]
    eager = [call(c, t) for c, t in variants]
    model.use_cuda_graph = True
    for rnd in range(2):                       # round 0 captures (2 shapes), round 1 replays
        for (c, t), ref in zip(variants, eager):
            out = call(c, t)
            assert torch.equal(out, ref), f"round {rnd}: graph replay differs from the host-launched step"
    assert model.graph_replays == 6 and len(model._graphs) == 2


def test_last_block_trim_is_exact():
    """The last single block computed on the current clip's rows only (trim_last_block) gives bit-identical velocities."""
    from oracle import flux_oracle as FO
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    kw = dict(num_layers=1, num_single_layers=2)
    cfg = FO.FluxConfig(**kw)
    dev = torch.device("cuda:0")
    params = FO.synthetic_flux_params(cfg, seed=5)
    g = torch.Generator().manual_seed(6)
    clips = [torch.randn(2, 16, 2, 12, 20, generator=g).bfloat16().to(dev), torch.randn(2, 16, 1, 24, 40, generator=g).bfloat16().to(dev),
             torch.randn(2, 16, 1, 48, 80, generator=g).bfloat16().to(dev)]
    enc = (torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().to(dev)
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[1, 50:] = 0
    mask = mask.to(dev)
    pooled = torch.randn(2, 768, generator=g).to(dev)
    t = torch.tensor([500.0, 500.0], device=dev)
    model = B200FluxTransformer(FluxConfigB200(**kw), params, device=dev)
    outs = []
    for trim in (False, True):
        model.trim_last_block = trim
        outs.append(model(sample=[clips], timestep_ratio=t, encoder_hidden_states=enc, encoder_attention_mask=mask,
                          pooled_projections=pooled)[0].float().cpu())
    plan = model.last_plan
    assert (plan.seq - plan.last_tokens) // 128 > 0, "shape too small to trim anything"
    assert torch.equal(outs[0], outs[1])
