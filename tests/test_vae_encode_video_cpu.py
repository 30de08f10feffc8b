"""Video encode without a GPU: the oracle's chunked / tiled encode against the reference's moments, the chunk schedule,
and the window_size check of B200CausalVAE.encode."""
import pytest
import torch

from oracle import vae_encode_oracle as VEO
from oracle import vae_oracle as VO


def _load(golden_dir):
    g = torch.load(golden_dir / "vae_encoder_video_small.pt", weights_only=False)
    cfg = VO.VaeEncoderConfig(**g["cfg"])
    return g, cfg, VO.synthetic_vae_params(cfg, seed=g["param_seed"])


def test_chunked_encode_oracle_matches_reference(golden_dir):
    g, cfg, p = _load(golden_dir)
    with torch.no_grad():
        whole = VO.encode_moments(p, cfg, g["clip"])
        assert whole.shape == g["whole"].shape == (1, 32, 4, 4, 6)
        assert (whole - g["whole"]).abs().max().item() < 1e-5
        for w in (8, 16):
            m = VEO.chunk_encode_moments(p, cfg, g["clip"], window_size=w)
            assert m.shape == g[f"chunk{w}"].shape == whole.shape
            assert (m - g[f"chunk{w}"]).abs().max().item() < 1e-5, w
    assert g["whole"].abs().mean().item() > 0.05


def test_tiled_encode_oracle_matches_reference(golden_dir):
    g, cfg, p = _load(golden_dir)
    with torch.no_grad():
        tiled = VEO.tiled_encode_moments(p, cfg, g["clip"], tile_sample_min_size=32)
        tiled_c = VEO.tiled_encode_moments(p, cfg, g["clip"], tile_sample_min_size=32, window_size=8)
    # 32-px tiles every 24 px of a 32 x 48 clip: 4-latent tiles cropped to 3, the edge tiles 1 (8 px) and 3 (24 px) wide
    assert tiled.shape == g["tiled32"].shape == tiled_c.shape == (1, 32, 4, 4, 6)
    assert (tiled - g["tiled32"]).abs().max().item() < 1e-5
    assert (tiled_c - g["tiled32_chunk8"]).abs().max().item() < 1e-5
    assert (tiled - g["whole"]).abs().max().item() > 1e-3      # tiling changes the latent, as in the reference


def test_chunk_schedule():
    from pyramid_flow_b200.vae import B200CausalVAE
    split = B200CausalVAE.chunk_frame_split
    assert split(25, 8) == [(0, 9), (9, 17), (17, 25)]
    assert split(121, 16) == [(0, 17)] + [(a, a + 16) for a in range(17, 113, 16)] + [(113, 121)]
    assert split(121, 16)[-2:] == [(97, 113), (113, 121)]
    assert split(1, 16) == [(0, 1)]
    assert split(9, 16) == [(0, 9)]              # the whole-clip path: one chunk
    assert split(25, 25) == [(0, 25)]


@pytest.mark.parametrize("window", [12, 0, -8, 4])
def test_window_must_be_a_multiple_of_the_temporal_downsampling(window):
    from pyramid_flow_b200.vae import B200CausalVAE, VaeConfigB200
    g = torch.Generator().manual_seed(0)
    cfg = VO.VaeEncoderConfig(**{"block_out_channels": (64, 128, 128, 128), "layers_per_block": (1, 2, 1, 1)})
    vae = B200CausalVAE(VaeConfigB200(enc_block_out_channels=cfg.block_out_channels,
                                      enc_layers_per_block=cfg.layers_per_block),
                        VO.synthetic_vae_params(cfg, seed=1), device="cpu")
    x = torch.randn(1, 3, 25, 32, 48, generator=g)
    with pytest.raises(ValueError, match="multiple of the temporal down-sampling factor 8"):
        vae.encode(x, temporal_chunk=True, window_size=window)
