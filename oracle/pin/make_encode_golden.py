"""Generate tests/golden/vae_encoder_video_small.pt: what the UNMODIFIED reference `CausalVideoVAE.encode` computes for a
25-frame clip through its video paths, pinning oracle/vae_encode_oracle.py.

    python oracle/pin/make_encode_golden.py      (CPU; needs a readable reference checkout, see oracle/pin/ref_shim.py)

The encoder is the tiny one of tests/golden/vae_encoder_small.pt (make_golden.py's VAE_ENC_SMALL, parameter seed 1); the
input is a 1 x 3 x 25 x 32 x 48 clip from torch.Generator().manual_seed(4).  Stored moments [1, 32, 4, 4, 6]:
`whole` (encode), `chunk8` / `chunk16` (temporal_chunk with window_size 8 / 16, chunk_encode V:311-341), and with
enable_tiling() and tile_sample_min_size=32 (tiled_encode V:409-466) `tiled32_chunk8` (window 8) and `tiled32` (unchunked).
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from oracle.pin.make_golden import GOLD, VAE_ENC_SMALL  # noqa: E402  (also installs the reference shim)


def main() -> None:
    from video_vae import CausalVideoVAE
    from oracle import vae_oracle as VO
    cfg = VO.VaeEncoderConfig(**VAE_ENC_SMALL)
    params = VO.synthetic_vae_params(cfg, seed=1)
    vae = CausalVideoVAE(encoder_out_channels=16, decoder_in_channels=16, encoder_block_out_channels=cfg.block_out_channels,
                         encoder_layers_per_block=cfg.layers_per_block, decoder_block_out_channels=(32, 32, 32, 32),
                         decoder_layers_per_block=(1, 1, 1, 1)).eval()
    sd = vae.state_dict()
    sd.update(params)
    vae.load_state_dict(sd, strict=True)
    clip = torch.randn(1, 3, 25, 32, 48, generator=torch.Generator().manual_seed(4))
    out = {"cfg": VAE_ENC_SMALL, "param_seed": 1, "clip": clip}
    with torch.no_grad():
        out["whole"] = vae.encode(clip).latent_dist.parameters
        for w in (8, 16):
            out[f"chunk{w}"] = vae.encode(clip, temporal_chunk=True, window_size=w).latent_dist.parameters
        vae.enable_tiling()
        out["tiled32_chunk8"] = vae.encode(clip, temporal_chunk=True, window_size=8,
                                           tile_sample_min_size=32).latent_dist.parameters
        out["tiled32"] = vae.encode(clip, tile_sample_min_size=32).latent_dist.parameters
    for k in ("chunk8", "chunk16"):
        print(f"[make_encode_golden] {k} vs whole max-abs {float((out[k] - out['whole']).abs().max()):.3e}")
    print("[make_encode_golden]", tuple(out["whole"].shape), tuple(out["tiled32"].shape), float(out["whole"].abs().mean()),
          "tiled chunk8 vs unchunked", float((out["tiled32_chunk8"] - out["tiled32"]).abs().max()))
    torch.save(out, GOLD / "vae_encoder_video_small.pt")


if __name__ == "__main__":
    main()
