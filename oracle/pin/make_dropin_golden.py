"""Generate tests/golden/dropin_reference.pt: what the UNMODIFIED reference pipeline computes WITH ITS OWN MODULES on the GPU
for the two calls of tests/test_dropin_gpu.py (bf16 weights under torch.autocast), so that the drop-in classes can be compared
with the original project where its sources are not available.

    python oracle/pin/make_dropin_golden.py      (needs a GPU and the reference staged by oracle/pin/stage_reference.py)

Stored: `generate_latents` fp32 [1, 16, T, h, w] (final latents of generate()), `i2v_frames` uint8 [frames, H/2, W/2, 3]
(every second pixel of generate_i2v()'s decoded frames), `device` (name of the GPU the reference ran on).
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
GOLD = ROOT / "tests" / "golden"


def main() -> None:
    from tests import test_dropin_gpu as T
    ref = T.load_reference()
    assert ref is not None, "reference packages not staged (oracle/pin/stage_reference.py)"
    dev = torch.device("cuda:0")
    g = torch.load(GOLD / "sampler_small.pt", weights_only=False)
    lat = T.run_generate(ref, T.reference_dit(ref, g, dev), g, dev)
    g2 = torch.load(GOLD / "sampler_i2v_small.pt", weights_only=False)
    frames = T.run_generate_i2v(ref, T.reference_dit(ref, g2, dev), T.reference_vae(ref, dev), g2, dev)
    out = {"generate_latents": lat, "i2v_frames": frames[:, ::2, ::2].to(torch.uint8).contiguous(),
           "device": torch.cuda.get_device_name(0)}
    torch.save(out, GOLD / "dropin_reference.pt")
    print(f"[make_dropin_golden] latents {tuple(lat.shape)} |mean| {lat.abs().mean():.3f}; frames {tuple(out['i2v_frames'].shape)} "
          f"std {frames.std():.1f} on {out['device']}")


if __name__ == "__main__":
    main()
