"""THE DROP-IN against the ORIGINAL project (INTEGRATION.md).  Two calls of the reference pipeline -- `generate()` to final
latents, and `generate_i2v()` with `output_type="pil"` (vae.encode for the image latent, decode_latent for the frames) -- on
fixed seeds, text embeddings and injected block noise, with

    pipe.dit = B200FluxTransformer(...)   and   pipe.vae = B200CausalVAE(...)

in place of the reference's modules.  What the reference computes with ITS OWN modules (bf16 weights under torch.autocast, the
README's way of running it) is stored in tests/golden/dropin_reference.pt (oracle/pin/make_dropin_golden.py ran the unmodified
reference on an H100), so the comparison with the original always runs:

  * always: the drop-in classes, driven by this repository's mirror of the pipeline loop (pyramid_flow_b200/sampler.py, itself
    pinned to the reference loop by tests/test_sampler_cpu.py), against the stored reference outputs;
  * where the reference's sources are staged (oracle/_ref, see oracle/pin/stage_reference.py): additionally the UNMODIFIED
    pipeline class `PyramidDiTForVideoGeneration` runs its own loop (P:706-788, 791-1003, 1006-1243) with the drop-in objects
    and with its own modules, and both are compared with each other and with the stored outputs."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def load_reference():
    """The reference's classes from the staged copy, or None where it is not staged."""
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        return None
    ref_shim.install()
    import diffusion_schedulers
    import pyramid_dit
    import video_vae
    return dict(pipeline=pyramid_dit.PyramidDiTForVideoGeneration,
                flux=__import__("pyramid_dit.flux_modules", fromlist=["PyramidFluxTransformer"]).PyramidFluxTransformer,
                sched=diffusion_schedulers.PyramidFlowMatchEulerDiscreteScheduler, vae=video_vae.CausalVideoVAE)


@pytest.fixture(scope="module")
def ref():
    return load_reference()


@pytest.fixture(scope="module")
def stored(golden_dir):
    return torch.load(golden_dir / "dropin_reference.pt", weights_only=False)


class _FakeText:
    """generate() asks for the prompt first, then for the negative prompt (P:1066-1067)."""

    def __init__(self, enc, mask, pooled):
        self.enc, self.mask, self.pooled, self.calls = enc, mask, pooled, 0

    def __call__(self, prompt, device):
        i = 1 if self.calls % 2 == 0 else 0
        self.calls += 1
        return self.enc[i:i + 1], self.mask[i:i + 1], self.pooled[i:i + 1]


def _make_pipe(ref, dit, vae, g, dev):
    pipe = object.__new__(ref["pipeline"])
    pipe.dit = dit
    pipe.vae = vae
    pipe.text_encoder = _FakeText(g["enc"].to(dev).bfloat16(), g["mask"].to(dev), g["pooled"].to(dev).bfloat16())
    pipe.scheduler = ref["sched"](shift=1.0, stages=3, stage_range=[0, 1 / 3, 2 / 3, 1], gamma=1 / 3)
    pipe.stages = [1, 2, 4]
    pipe.frame_per_unit = 1
    pipe.model_name = "pyramid_flux"
    pipe.sequential_offload_enabled = False
    pipe.downsample = 8
    pipe.vae_shift_factor, pipe.vae_scale_factor = -0.04, 1 / 1.8726
    pipe.vae_video_shift_factor, pipe.vae_video_scale_factor = -0.2343, 1 / 3.0986
    noises = [n.clone() for n in g["noises"]]
    pipe.sample_block_noise = lambda bs, ch, temp, height, width: noises.pop(0)
    return pipe


def _flux_params(g):
    from oracle import flux_oracle as FO
    return FO.synthetic_flux_params(FO.FluxConfig(**g["cfg"]), seed=g["param_seed"])


def reference_dit(ref, g, dev):
    dit = ref["flux"](**g["cfg"]).eval()
    dit.load_state_dict(_flux_params(g), strict=True)
    return dit.to(dev, torch.bfloat16)


def dropin_dit(g, dev):
    """The drop-in DiT on the weights the reference module holds (bf16), without needing the reference class."""
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    return B200FluxTransformer(FluxConfigB200(**g["cfg"]), {k: v.bfloat16() for k, v in _flux_params(g).items()}, device=dev)


# a small VAE with non-degenerate weights (decoder: the small golden config; encoder likewise); every tensor of the reference
# VAE's state dict is set from a seed
VAE_BLOCKS, VAE_LAYERS = (64, 64, 128, 128), (1, 1, 1, 1)


def _vae_params():
    from oracle import vae_oracle as VO
    dcfg = VO.VaeDecoderConfig(block_out_channels=VAE_BLOCKS, layers_per_block=VAE_LAYERS)
    ecfg = VO.VaeEncoderConfig(block_out_channels=VAE_BLOCKS, layers_per_block=VAE_LAYERS)
    new = {**VO.synthetic_vae_params(dcfg, seed=4), **VO.synthetic_vae_params(ecfg, seed=5)}
    # latent_dist.sample() draws from the global RNG (D:381-389): pin log-variance at -30 so the image latent is its mean
    new["quant_conv.conv.weight"][16:] = 0
    new["quant_conv.conv.bias"][16:] = -30.0
    return new


def reference_vae(ref, dev):
    rvae = ref["vae"](encoder_out_channels=16, decoder_in_channels=16, encoder_block_out_channels=VAE_BLOCKS,
                      encoder_layers_per_block=VAE_LAYERS, decoder_block_out_channels=VAE_BLOCKS,
                      decoder_layers_per_block=VAE_LAYERS).eval()
    new = _vae_params()
    assert set(new) == set(rvae.state_dict())
    rvae.load_state_dict(new, strict=True)
    rvae = rvae.to(dev, torch.bfloat16)
    rvae.enable_tiling()
    return rvae


def dropin_vae(dev):
    from pyramid_flow_b200.vae import B200CausalVAE, VaeConfigB200
    cfg = VaeConfigB200(block_out_channels=VAE_BLOCKS, layers_per_block=VAE_LAYERS, enc_block_out_channels=VAE_BLOCKS,
                        enc_layers_per_block=VAE_LAYERS)
    vae = B200CausalVAE(cfg, {k: v.bfloat16() for k, v in _vae_params().items()}, device=dev)
    vae.enable_tiling()
    return vae


def _image_u8(g):
    return (g["image_tensor"][0, :, 0].permute(1, 2, 0) * 127.5 + 127.5).round().clamp(0, 255).byte()


def run_generate(ref, dit, g, dev):
    """The unmodified pipeline's generate() around `dit` -> final latents, fp32 on the host."""
    pipe = _make_pipe(ref, dit, None, g, dev)
    gen = torch.Generator().manual_seed(g["latent_seed"])
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        lat = pipe.generate(prompt="x", generator=gen, output_type="latent", save_memory=True, **g["args"])
    torch.cuda.synchronize()
    return lat.float().cpu()


def run_generate_i2v(ref, dit, vae, g, dev):
    """The unmodified pipeline's generate_i2v(output_type="pil") around `dit` and `vae` -> frames [T, H, W, 3] as float."""
    import numpy as np
    from PIL import Image
    pipe = _make_pipe(ref, dit, vae, g, dev)
    gen = torch.Generator().manual_seed(g["latent_seed"])
    args = {k: v for k, v in g["args"].items() if k not in ("height", "width")}
    torch.manual_seed(123)                       # latent_dist.sample() draws from the global CUDA RNG (D:381-389)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        out = pipe.generate_i2v(prompt="x", input_image=Image.fromarray(_image_u8(g).numpy()), generator=gen,
                                output_type="pil", save_memory=True, **args)
    torch.cuda.synchronize()
    return torch.from_numpy(np.stack([np.asarray(f) for f in out])).float()


def _mirror(dit, vae, g):
    from pyramid_flow_b200.sampler import B200PyramidSampler
    from pyramid_flow_b200.scheduler import B200FlowMatchScheduler
    noises = [n.clone() for n in g["noises"]]
    return B200PyramidSampler(dit, B200FlowMatchScheduler(), vae=vae, block_noise_fn=lambda *a: noises.pop(0))


def _rel_mse(a, b):
    return (((a - b) ** 2).mean() / (b ** 2).mean()).item()


def _frame_report(what, a, b):
    diff = (a - b).abs()
    print(f"{what}, uint8 frames {tuple(a.shape)}: mean |diff| {diff.mean():.3f} / 255, "
          f"99.9th pct {diff.flatten().kthvalue(int(0.999 * diff.numel())).values.item():.0f}, max {diff.max():.0f}; frame std {b.std():.1f}")
    return diff.mean().item()


def test_unmodified_generate_with_swapped_dit(ref, stored, golden_dir):
    dev = torch.device("cuda:0")
    g = torch.load(golden_dir / "sampler_small.pt", weights_only=False)
    ref_lat = stored["generate_latents"]
    assert ref_lat.shape == g["latents"].shape and ref_lat.abs().mean().item() > 1.0
    ours = dropin_dit(g, dev)
    enc, mask, pooled = g["enc"].to(dev).bfloat16(), g["mask"].to(dev), g["pooled"].to(dev).bfloat16()
    lat = _mirror(ours, None, g).generate(enc, mask, pooled, generator=torch.Generator().manual_seed(g["latent_seed"]),
                                          output_type="latent", **g["args"]).float().cpu()
    r_mirror = _rel_mse(lat, ref_lat)
    print(f"generate() final latents, drop-in (mirror loop) vs the stored output of the reference's own modules ({stored['device']}, "
          f"bf16): relative MSE {r_mirror:.3e}; |latent| mean {ref_lat.abs().mean():.3f}")
    assert r_mirror < 1e-3
    if ref is None:
        return
    # the unmodified pipeline, with its own module and with the drop-in built from it
    from pyramid_flow_b200.dit import B200FluxTransformer
    rdit = reference_dit(ref, g, dev)
    swapped = B200FluxTransformer.from_reference(rdit, device=dev)
    assert swapped.config.in_channels == rdit.config.in_channels and next(swapped.parameters()).device == next(rdit.parameters()).device
    outs = {"reference": run_generate(ref, rdit, g, dev), "b200": run_generate(ref, swapped, g, dev)}
    gold = g["latents"]
    r_pair = _rel_mse(outs["b200"], outs["reference"])
    r_ref, r_ours = _rel_mse(outs["reference"], gold), _rel_mse(outs["b200"], gold)
    print(f"unmodified pipeline: drop-in vs the reference's own modules on the same GPU (both bf16): relative MSE {r_pair:.3e}; "
          f"drop-in vs stored {_rel_mse(outs['b200'], ref_lat):.3e}; reference now vs stored {_rel_mse(outs['reference'], ref_lat):.3e}.  "
          f"(vs the CPU fp32 golden: reference {r_ref:.3e}, drop-in {r_ours:.3e} -- not comparable: on the GPU the pipeline draws its "
          f"start noise in bf16, a different random stream than the fp32 CPU run)")
    assert r_pair < 1e-3 and outs["reference"].abs().mean().item() > 1.0
    assert _rel_mse(outs["b200"], ref_lat) < 1e-3
    assert abs(r_ours - r_ref) < 0.05 * r_ref + 1e-3, "both runs must sit at the same distance from the fp32 CPU run"


def test_unmodified_generate_i2v_and_decode_latent_with_swapped_vae(ref, stored, golden_dir):
    """generate_i2v() needs vae.encode (image latent, P:911) and, with output_type='pil', decode_latent (P:1221-1243): the
    whole call runs on the drop-in objects; frames are compared as uint8 images with the reference modules' frames."""
    dev = torch.device("cuda:0")
    g = torch.load(golden_dir / "sampler_i2v_small.pt", weights_only=False)
    ref_frames = stored["i2v_frames"].float()           # every second pixel of the reference's frames
    n_frames = 1 + 8 * (g["args"]["temp"] - 1)
    assert ref_frames.shape == (n_frames, g["args"]["height"] // 2, g["args"]["width"] // 2, 3) and ref_frames.std().item() > 5.0
    odit, ovae = dropin_dit(g, dev), dropin_vae(dev)
    image = (_image_u8(g).float() / 255.0 - 0.5) / 0.5                       # ToTensor + Normalize(0.5, 0.5), P:907-910
    image = image.permute(2, 0, 1)[None, :, None].to(dev)
    enc, mask, pooled = g["enc"].to(dev).bfloat16(), g["mask"].to(dev), g["pooled"].to(dev).bfloat16()
    args = {k: v for k, v in g["args"].items()}
    torch.manual_seed(123)
    frames = _mirror(odit, ovae, g).generate_i2v(image, enc, mask, pooled, generator=torch.Generator().manual_seed(g["latent_seed"]),
                                                 output_type="pil", save_memory=True, **args).float().cpu()
    assert frames.shape[0] == n_frames
    assert _frame_report("generate_i2v -> decode_latent, drop-in (mirror loop) vs stored reference", frames[:, ::2, ::2], ref_frames) < 2.0
    if ref is None:
        return
    from pyramid_flow_b200.dit import B200FluxTransformer
    from pyramid_flow_b200.vae import B200CausalVAE
    rdit, rvae = reference_dit(ref, g, dev), reference_vae(ref, dev)
    svae = B200CausalVAE.from_reference(rvae, device=dev)
    svae.enable_tiling()
    a = run_generate_i2v(ref, B200FluxTransformer.from_reference(rdit, device=dev), svae, g, dev)
    b = run_generate_i2v(ref, rdit, rvae, g, dev)
    assert a.shape == b.shape and a.shape[0] == n_frames
    assert _frame_report("unmodified pipeline: drop-in vs the reference's own modules", a, b) < 2.0 and b.std().item() > 5.0
    assert _frame_report("unmodified pipeline: drop-in vs stored reference", a[:, ::2, ::2], ref_frames) < 2.0
