"""Video encode on the H100: temporal chunking and spatial tiling of B200CausalVAE.encode (chunk_encode / tiled_encode,
V:311-345 / V:409-466).  Chunking must reproduce the whole-clip moments bit for bit (GroupNorm statistics are per frame
and the conv's K order does not depend on how many frames a call holds); chunked and tiled moments are held to the
reference's moments and to the oracle with the bounds of test_vae_gpu.test_vae_encoder_matches_reference_golden."""
import gc

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
# torch.cuda.max_memory_allocated of tools/vae_encode_bench.py (121 x 768 x 1280 bf16 clip, full-size synthetic encoder,
# window 16, weights and clip resident), measured on an H100 80GB HBM3 at a 700 W power limit
BENCH_PEAK_GIB = {"chunked": 17.80, "tiled": 2.04}


def _small(golden_dir):
    from oracle import vae_oracle as VO
    from pyramid_flow_b200.vae import B200CausalVAE, VaeConfigB200
    g = torch.load(golden_dir / "vae_encoder_video_small.pt", weights_only=False)
    ecfg = VO.VaeEncoderConfig(**g["cfg"])
    params = VO.synthetic_vae_params(ecfg, seed=g["param_seed"])
    vae = B200CausalVAE(VaeConfigB200(enc_block_out_channels=ecfg.block_out_channels,
                                      enc_layers_per_block=ecfg.layers_per_block), params, device=DEV)
    return g, ecfg, params, vae


def _moments(vae, x, tiled=False, **kw):
    vae.enable_tiling(tiled)
    m = vae.encode(x.to(DEV), **kw).latent_dist.parameters
    torch.cuda.synchronize()
    return m


def test_chunked_encode_is_exact(golden_dir):
    g, _, _, vae = _small(golden_dir)
    x = g["clip"].bfloat16()
    whole = _moments(vae, x)
    assert whole.shape == (1, 32, 4, 4, 6)
    for w in (8, 16):
        assert torch.equal(_moments(vae, x, temporal_chunk=True, window_size=w), whole), w
    # batch 2 with different samples: every sample is its own clip with its own caches
    x2 = torch.cat([x, torch.randn(x.shape, generator=torch.Generator().manual_seed(9)).bfloat16()], 0)
    whole2 = _moments(vae, x2)
    assert torch.equal(whole2[:1], whole) and not torch.equal(whole2[1], whole2[0])
    assert torch.equal(_moments(vae, x2, temporal_chunk=True, window_size=8), whole2)
    # the 1-frame image and a clip shorter than one window take the one-chunk path
    assert torch.equal(_moments(vae, x[:, :, :1], temporal_chunk=True, window_size=8), _moments(vae, x[:, :, :1]))
    assert torch.equal(_moments(vae, x[:, :, :9], temporal_chunk=True, window_size=16), _moments(vae, x[:, :, :9]))


def test_tiled_chunked_encode_is_exact(golden_dir):
    g, _, _, vae = _small(golden_dir)
    x = g["clip"].bfloat16()
    tiled = _moments(vae, x, tiled=True, tile_sample_min_size=32)
    assert tiled.shape == (1, 32, 4, 4, 6)
    assert not torch.equal(tiled, _moments(vae, x))
    for w in (8, 16):
        assert torch.equal(_moments(vae, x, tiled=True, temporal_chunk=True, window_size=w, tile_sample_min_size=32), tiled), w
    # no tiling when the clip fits in one tile, as in the reference (V:293)
    assert torch.equal(_moments(vae, x, tiled=True, tile_sample_min_size=48), _moments(vae, x))


@pytest.mark.parametrize("case", ["chunk8", "chunk16", "tiled32", "tiled32_chunk8"])
def test_video_encode_matches_reference_golden(golden_dir, case):
    from oracle import vae_encode_oracle as VEO
    g, ecfg, params, vae = _small(golden_dir)
    x = g["clip"].bfloat16()                          # the VAE dtype; the reference ran on the un-rounded fp32 clip
    window = 16 if case == "chunk16" else 8 if case.endswith("8") else None
    tiled = case.startswith("tiled")
    kw = dict(temporal_chunk=window is not None, window_size=window or 16, tile_sample_min_size=32)
    ours = _moments(vae, x, tiled=tiled, **kw).float().cpu()
    pd = {k: v.to(DEV) for k, v in params.items()}

    def oracle(p, xx):
        if tiled:
            return VEO.tiled_encode_moments(p, ecfg, xx, tile_sample_min_size=32, window_size=window)
        return VEO.chunk_encode_moments(p, ecfg, xx, window_size=window)

    with torch.no_grad():
        ref = oracle(params, x.float())
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ref_bf16 = oracle(pd, x.to(DEV)).float().cpu()
    err = (ours - ref).abs().max().item()
    err_gold = (ours - g[case]).abs().max().item()
    err_pol = (ref_bf16 - ref).abs().max().item()
    print(f"vae encode {case}: max_abs vs oracle {err:.3e}, vs reference golden {err_gold:.3e}, "
          f"reference bf16 policy {err_pol:.3e}, |ref| mean {ref.abs().mean():.3f}")
    assert ours.shape == ref.shape == g[case].shape
    assert err < 5e-2 and err_gold < 6e-2 and err <= max(1.5 * err_pol, 1e-2)


def test_encode_edge_shapes_conv_kernel():
    """The shapes only chunked / tiled encode gives the strided conv: a later chunk's last temporal down-sampling (one
    output frame from 3 input frames, the first of them the cached one), and the 8-px edge tile (one output column)."""
    from pyramid_flow_b200.vae import B200CausalVAE, _Conv
    torch.manual_seed(2)
    holder = B200CausalVAE.__new__(B200CausalVAE)
    cases = [((2, 1, 1), 512, 512, 1, 12, 20), ((2, 1, 1), 128, 128, 1, 1, 1), ((2, 1, 1), 256, 256, 4, 2, 1),
             ((1, 2, 2), 128, 128, 8, 16, 1), ((1, 2, 2), 256, 256, 4, 1, 1), ((1, 2, 2), 64, 64, 2, 1, 3)]
    for (stride, ci, co, t_out, h_out, w_out) in cases:
        st, sh, sw = stride
        wt = (torch.randn(co, ci, 3, 3, 3) * (ci * 27) ** -0.5).bfloat16().float()
        bias = torch.randn(co) * 0.1
        cv = _Conv({"c.conv.weight": wt, "c.conv.bias": bias}, "c", DEV)
        cv.stride = stride
        t_in = (t_out - 1) * st + 3                   # the conv's whole input, halo frames included
        xin = torch.randn(t_in + 1, h_out * sh, w_out * sw, ci, device=DEV).bfloat16()
        xv = xin[1:]                                  # offset by one frame, as a later chunk's stride-2 input is
        ref = F.conv3d(F.pad(xv.permute(3, 0, 1, 2)[None].float(), (1, 1, 1, 1, 0, 0)), wt.to(DEV), bias.to(DEV),
                       stride=stride)[0].permute(1, 2, 3, 0)
        assert tuple(ref.shape) == (t_out, h_out, w_out, co)
        out = torch.zeros(t_out, h_out, w_out, co, device=DEV, dtype=torch.bfloat16)
        B200CausalVAE._conv(holder, cv, xv, t_out, h_out, w_out, out=out)
        torch.cuda.synchronize()
        err = (out.float() - ref).abs().max().item()
        assert err < 3e-2, (stride, ci, co, t_out, h_out, w_out, err)


@pytest.fixture(scope="module")
def full_size():
    from oracle import vae_oracle as VO
    from pyramid_flow_b200.vae import B200CausalVAE, VaeConfigB200
    ecfg = VO.VaeEncoderConfig()
    vae = B200CausalVAE(VaeConfigB200(enc_block_out_channels=ecfg.block_out_channels,
                                      enc_layers_per_block=ecfg.layers_per_block),
                        VO.synthetic_vae_params(ecfg, seed=0), device=DEV)
    yield vae
    del vae
    gc.collect()
    torch.cuda.empty_cache()


def _clip(frames, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(1, 3, frames, 768, 1280, generator=g, device=DEV, dtype=torch.bfloat16)


def test_full_size_chunked_encode_is_exact(full_size):
    x = _clip(25)
    whole = _moments(full_size, x)
    chunked = _moments(full_size, x, temporal_chunk=True, window_size=8)
    assert whole.shape == (1, 32, 4, 96, 160) and bool(torch.isfinite(whole).all())
    assert torch.equal(chunked, whole), (chunked.float() - whole.float()).abs().max().item()


@pytest.mark.parametrize("mode", ["chunked", "tiled"])
def test_full_size_121_frames(full_size, mode):
    x = _clip(121)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m = _moments(full_size, x, tiled=mode == "tiled", temporal_chunk=True, window_size=16, tile_sample_min_size=256)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"vae encode 121 x 768 x 1280 {mode}: peak allocated {peak:.2f} GiB (bench {BENCH_PEAK_GIB[mode]:.2f} GiB)")
    assert m.shape == (1, 32, 16, 96, 160)
    assert bool(torch.isfinite(m).all())
    assert peak < 1.3 * BENCH_PEAK_GIB[mode]
