"""Loop-level parity on an H100: the sampler mirror driving the CUDA DiT vs the same loop driving the fp32 oracle
(identical start noise, injected block noise and text embeddings) -> final-latent error (BASELINE.json north_star)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_generate_latents_match_oracle_loop(golden_dir):
    from oracle import flux_oracle as FO
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    from pyramid_flow_b200.sampler import B200PyramidSampler
    from pyramid_flow_b200.scheduler import B200FlowMatchScheduler
    from tests.test_sampler_cpu import OracleDit

    g = torch.load(golden_dir / "sampler_small.pt", weights_only=False)
    cfg = FO.FluxConfig(**g["cfg"])
    params = FO.synthetic_flux_params(cfg, seed=g["param_seed"])
    dev = torch.device("cuda:0")
    enc, mask, pooled = g["enc"].to(dev), g["mask"].to(dev), g["pooled"].to(dev)

    def run(dit, dtype):
        noises = [n.clone() for n in g["noises"]]
        s = B200PyramidSampler(dit, B200FlowMatchScheduler(), block_noise_fn=lambda *a: noises.pop(0))
        gen = torch.Generator().manual_seed(g["latent_seed"])
        lat0 = torch.randn(1, 16, 4, 16, 16, generator=gen).to(dev)
        out = s.generate(enc.to(dtype), mask, pooled.to(dtype), output_type="latent", latents=lat0.to(dtype), **g["args"])
        return out.float().cpu(), s

    ref, _ = run(OracleDit(cfg, {k: v.to(dev) for k, v in params.items()}), torch.float32)
    # the oracle loop on the GPU reproduces the reference's CPU golden (same loop, fp32)
    assert (ref - g["latents"]).abs().max().item() < 2e-3
    ours, s = run(B200FluxTransformer(FluxConfigB200(**g["cfg"]), params, device=dev), torch.bfloat16)
    torch.cuda.synchronize()
    err = (ours - ref).abs().max().item()
    mse = ((ours - ref) ** 2).mean().item()
    rel = mse / (ref ** 2).mean().item()
    print(f"sampler loop ({s.dit_calls} DiT calls, bf16 latents): final-latent max_abs {err:.3e} mse {mse:.3e} relative mse {rel:.3e} |ref| mean {ref.abs().mean():.3f}")
    # latents are O(3.7) here (2 steps per stage): bf16 latent storage alone costs 2^-9 relative per Euler step
    assert rel < 1e-3 and err < 0.5
