"""Video VAE encode at training-latent size: B200CausalVAE.encode on a 121 x 768 x 1280 clip, chunked and tiled.

    python tools/vae_encode_bench.py [--frames 121] [--height 768] [--width 1280] [--window 16] [--tile 256]
                                     [--warmup 1] [--rounds 3] [--reference] [--ref-rounds 1] [--json out.json]

The encoder has the full-size configuration (128/256/512/512 channels, 2 layers per block) with the seeded synthetic
weights of oracle.vae_oracle.synthetic_vae_params, and the clip is a seeded bf16 tensor.  Two modes:
  chunked: encode(x, temporal_chunk=True, window_size=16), untiled;
  tiled:   the same after enable_tiling(), with tile_sample_min_size=256.
Each mode is warmed up, then timed `rounds` times (CUDA events around one encode, median reported), with
torch.cuda.max_memory_allocated over the timed rounds (the weights and the input clip are resident).

--reference also runs the unmodified reference `CausalVideoVAE.encode` (the copy staged under oracle/_ref by build()),
with the same weights cast to bf16, the same clip and the same arguments, and reports its time, its peak memory and the
relative RMS difference of the two implementations' moments.  The card's name, power limit and max SM clock are read with
nvidia-smi (a query only) in the same run.
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from oracle import vae_oracle as VO  # noqa: E402
from pyramid_flow_b200 import _lib  # noqa: E402
from pyramid_flow_b200.vae import B200CausalVAE, VaeConfigB200  # noqa: E402

MODES = ("chunked", "tiled")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": out or "unavailable"}


def full_size_encoder(dev):
    """The full-size encoder (VaeEncoderConfig defaults) with synthetic weights: (oracle config, fp32 params, ours)."""
    ecfg = VO.VaeEncoderConfig()
    params = VO.synthetic_vae_params(ecfg, seed=0)
    vae = B200CausalVAE(VaeConfigB200(enc_block_out_channels=ecfg.block_out_channels,
                                      enc_layers_per_block=ecfg.layers_per_block), params, device=dev)
    return ecfg, params, vae


def seeded_clip(frames, height, width, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(1, 3, frames, height, width, generator=g, device=dev, dtype=torch.bfloat16)


def run_encode(vae, x, mode, window, tile):
    """One encode in `mode` (works for ours and for the reference: both have enable_tiling / disable_tiling)."""
    if mode == "tiled":
        vae.enable_tiling()
    else:
        vae.disable_tiling()
    with torch.no_grad():
        return vae.encode(x, temporal_chunk=True, window_size=window, tile_sample_min_size=tile).latent_dist.parameters


def time_mode(fn, warmup, rounds):
    """(median ms, per-round ms, peak bytes over the timed rounds, last output)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times, peak, out = [], 0, None
    for _ in range(rounds):
        out = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        peak = max(peak, torch.cuda.max_memory_allocated())
    return statistics.median(times), times, peak, out


def reference_encoder(params, dev):
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        sys.exit("--reference: the reference packages are not staged under oracle/_ref (build() stages them)")
    ref_shim.install()
    from video_vae import CausalVideoVAE
    ref = CausalVideoVAE(encoder_out_channels=16, decoder_in_channels=16).eval()
    sd = ref.state_dict()
    sd.update(params)
    ref.load_state_dict(sd, strict=True)
    del ref.decoder, ref.post_quant_conv                 # encode does not use them
    return ref.to(device=dev, dtype=torch.bfloat16)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=121)
    ap.add_argument("--height", type=int, default=768)
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--window", type=int, default=16)
    ap.add_argument("--tile", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reference", action="store_true", help="also time the unmodified reference encode (eager, bf16)")
    ap.add_argument("--ref-rounds", type=int, default=1)
    ap.add_argument("--json", type=str, default=None, help="also write the result line to this file")
    args = ap.parse_args()

    _lib.require_device()
    dev = torch.device("cuda:0")
    info = card()
    _, params, vae = full_size_encoder(dev)
    x = seeded_clip(args.frames, args.height, args.width, dev)
    res = {"tool": "vae_encode_bench", "card": info, "clip": [1, 3, args.frames, args.height, args.width],
           "window_size": args.window, "tile_sample_min_size": args.tile, "warmup": args.warmup, "rounds": args.rounds,
           "modes": {}}
    ours = {}
    for mode in MODES:
        ms, times, peak, out = time_mode(lambda: run_encode(vae, x, mode, args.window, args.tile), args.warmup, args.rounds)
        ours[mode] = out.float().cpu()
        res["modes"][mode] = {"ms_per_clip": ms, "round_ms": times, "frames_per_s": args.frames / (ms / 1e3),
                              "peak_alloc_gib": peak / 2 ** 30, "moments_shape": list(out.shape),
                              "finite": bool(torch.isfinite(out).all())}
        print(f"[vae_encode_bench] ours {mode}: {ms:.1f} ms/clip ({args.frames / (ms / 1e3):.1f} frames/s), "
              f"peak {peak / 2 ** 30:.2f} GiB, moments {tuple(out.shape)}", flush=True)
        del out
    if args.reference:
        del vae
        torch.cuda.empty_cache()
        ref = reference_encoder(params, dev)
        for mode in MODES:
            ms, times, peak, out = time_mode(lambda: run_encode(ref, x, mode, args.window, args.tile), 1, args.ref_rounds)
            r = out.float().cpu()
            rel = ((ours[mode] - r).pow(2).mean().sqrt() / r.pow(2).mean().sqrt()).item()
            m = res["modes"][mode]
            m["reference"] = {"ms_per_clip": ms, "round_ms": times, "frames_per_s": args.frames / (ms / 1e3),
                              "peak_alloc_gib": peak / 2 ** 30, "moments_rel_rms_diff": rel}
            m["speedup_vs_reference"] = ms / m["ms_per_clip"]
            print(f"[vae_encode_bench] reference {mode}: {ms:.1f} ms/clip, peak {peak / 2 ** 30:.2f} GiB; ours is "
                  f"{m['speedup_vs_reference']:.2f}x faster; moments relative RMS difference {rel:.3e}", flush=True)
            del out
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
