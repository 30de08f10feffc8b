"""End-to-end generate() + decode on one or N GPUs with synthetic text embeddings and random-init weights:
python tools/e2e_generate.py [--height 768 --width 1280 --temp 31]   (BASELINE configs[2]; --temp 16 --height 384 --width 640 = configs[1])
torchrun --nproc-per-node N tools/e2e_generate.py ...   : every rank runs the same sampler loop (same seeds); the DiT step is
sharded CFG x sequence-parallel (sp.py) and the VAE decode is context-parallel (temporal split + halo exchange).
Reports wall-clock frames/s (excluding text encoding) and aggregate DiT token-passes/s."""
import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch

from bench import random_flux_state_dict, random_vae_state_dict
from pyramid_flow_b200.dit import B200FluxTransformer
from pyramid_flow_b200.sampler import B200PyramidSampler
from pyramid_flow_b200.scheduler import B200FlowMatchScheduler
from pyramid_flow_b200.vae import B200CausalVAE, VaeConfigB200

ap = argparse.ArgumentParser()
ap.add_argument("--height", type=int, default=768)
ap.add_argument("--width", type=int, default=1280)
ap.add_argument("--temp", type=int, default=31)
ap.add_argument("--no-decode", action="store_true")
ap.add_argument("--graph", action="store_true", help="capture every (unit, stage) step shape into a CUDA graph (pays ~30 ms per shape; useful on slow hosts)")
ap.add_argument("--window", type=int, default=4, help="latent frames per VAE chunk (exact; memory knob)")
args = ap.parse_args()
import os
world, rank, local = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=dev)
torch.manual_seed(1234)          # block noise comes from the global CPU RNG: identical on every rank
cfg, sd = random_flux_state_dict(dict(num_layers=8, num_single_layers=16), dev, seed=0)
dit = B200FluxTransformer(cfg, sd, device=dev)
del sd
vae = None
if not args.no_decode:
    vae = B200CausalVAE(VaeConfigB200(), random_vae_state_dict(dev), device=dev)
g = torch.Generator().manual_seed(0)
enc = (torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().to(dev)
mask = torch.ones(2, 128, dtype=torch.long, device=dev)
pooled = torch.randn(2, 768, generator=g).bfloat16().to(dev)

tokens = [0]
orig = dit.forward


def counting(*a, **k):
    out = orig(*a, **k)
    tokens[0] += 2 * dit.last_plan.seq
    return out


if world > 1:
    from pyramid_flow_b200 import sp as SP
    dit.set_parallel_layout(SP.make_layout())
    if vae is not None:
        vae.set_context_parallel(None)
dit.forward = counting
dit.use_cuda_graph = args.graph   # each (unit, stage) shape lives for 10-20 steps only: capture pays off on slow hosts
sampler = B200PyramidSampler(dit, B200FlowMatchScheduler(), vae=vae)
torch.cuda.synchronize()
t0 = time.time()
lat = sampler.generate(enc, mask, pooled, height=args.height, width=args.width, temp=args.temp,
                       num_inference_steps=[20, 20, 20], video_num_inference_steps=[10, 10, 10], guidance_scale=7.0,
                       video_guidance_scale=5.0, generator=torch.Generator().manual_seed(1), output_type="latent")
torch.cuda.synchronize()
t1 = time.time()
frames = 1 + 8 * (args.temp - 1)
res = {"config": f"miniFLUX {args.height}x{args.width}, temp={args.temp} ({frames} frames), steps 20/10, guidance 7/5, {world} GPU(s), bf16",
       "dit_calls": sampler.dit_calls, "dit_seconds": t1 - t0, "dit_token_passes": tokens[0],
       "dit_token_passes_per_s": tokens[0] / (t1 - t0), "latent_finite": bool(torch.isfinite(lat.float()).all())}
if vae is not None:
    lat = torch.nan_to_num(lat.float()).clamp(-4, 4).to(lat.dtype)    # random weights: keep the decoder input sane
    u8 = None
    t2 = time.time()
    # un-tiled, temporally chunked decode (exact); window is a memory knob
    lat_n = lat.clone()
    lat_n[:, :, :1] = lat_n[:, :, :1] / sampler.vae_scale_factor + sampler.vae_shift_factor
    if lat_n.shape[2] > 1:
        lat_n[:, :, 1:] = lat_n[:, :, 1:] / sampler.vae_video_scale_factor + sampler.vae_video_shift_factor
    img = vae.decode(lat_n, temporal_chunk=True, window_size=args.window).sample
    u8 = img.float().mul(127.5).add(127.5).clamp(0, 255).byte().permute(0, 2, 3, 4, 1).contiguous().cpu()
    torch.cuda.synchronize()
    t3 = time.time()
    res.update(decode_seconds=t3 - t2, video_shape=list(u8.shape), frames_per_s_end_to_end=frames / ((t1 - t0) + (t3 - t2)),
               decode_frames_per_s=frames / (t3 - t2), peak_mem_gib=torch.cuda.max_memory_allocated() / 2 ** 30)
if world > 1:
    dist.barrier()
if rank == 0:
    print(json.dumps(res))
if world > 1:
    dist.destroy_process_group()
