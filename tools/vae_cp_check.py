"""torchrun --nproc-per-node N tools/vae_cp_check.py : context-parallel VAE decode (temporal split + per-conv halo
exchange) equals the single-GPU decode bit for bit, and is timed against it.  Run on a node with N = 2, 4 or 8."""
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch
import torch.distributed as dist

from bench import random_vae_state_dict
from pyramid_flow_b200.vae import B200CausalVAE, VaeConfigB200

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
vae = B200CausalVAE(VaeConfigB200(), random_vae_state_dict(dev), device=dev)


def timed(fn):
    fn()
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1)], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return out, t.item()


cases = [(1 + 2 * world, 24, 40, 2), (2 + 5 * world, 24, 40, 2), (int(os.environ.get("PF_CP_T", "31")), 96, 160, 2)]
for (T, h, w, win) in cases:
    g = torch.Generator().manual_seed(5)
    z = torch.randn(1, 16, T, h, w, generator=g).bfloat16().to(dev)
    vae.set_context_parallel(None)
    vae._cp = None
    ref, ms1 = timed(lambda: vae.decode(z, temporal_chunk=True, window_size=win).sample)
    vae.set_context_parallel(None)          # default group: all ranks
    out, msn = timed(lambda: vae.decode(z, temporal_chunk=True, window_size=win).sample)
    same = bool(torch.equal(out, ref))
    err = (out.float() - ref.float()).abs().max().item()
    flags = [None] * world
    dist.all_gather_object(flags, (same, err))
    if rank == 0:
        fr = ref.shape[2]
        print(f"[vae_cp_check] latent {T}x{h}x{w} -> {tuple(ref.shape)}: 1 GPU (chunked, window {win}) {ms1:.1f} ms = "
              f"{fr / ms1 * 1e3:.1f} frames/s | {world} GPUs context-parallel {msn:.1f} ms = {fr / msn * 1e3:.1f} frames/s "
              f"(x{ms1 / msn:.2f}); {len(vae.cp_frame_split(T, world, vae.cp_frames_per_round))} round(s) of {vae.cp_frames_per_round} latent frames per rank, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB; bit-identical per rank {[f[0] for f in flags]} "
              f"max|diff| {max(f[1] for f in flags):.2e}", flush=True)
    assert err < 1e-3, err
dist.destroy_process_group()
