"""torchrun --nproc-per-node N tools/sp_check.py : the CFG x SP parallel DiT step equals the single-GPU step (same kernels,
same inputs); run on a node with N = 2, 4 or 8."""
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch
import torch.distributed as dist

from oracle import flux_oracle as FO
from pyramid_flow_b200 import sp as SP
from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
lay = SP.make_layout()

for name, kw, clip_shapes, tlen in [
    ("small D=256", dict(num_layers=2, num_single_layers=2, num_attention_heads=4, attention_head_dim=64, in_channels=64,
                         joint_attention_dim=128, pooled_projection_dim=64),
     [(2, 16, 2, 4, 8), (2, 16, 1, 8, 16), (2, 16, 1, 16, 32)], 24),
    ("miniFLUX width, 30 heads", dict(num_layers=1, num_single_layers=2),
     [(2, 16, 2, 12, 20), (2, 16, 1, 24, 40), (2, 16, 1, 48, 80)], 128),
]:
    cfg = FO.FluxConfig(**kw)
    params = FO.synthetic_flux_params(cfg, seed=0)
    g = torch.Generator().manual_seed(1)
    clips = [torch.randn(s, generator=g).bfloat16().to(dev) for s in clip_shapes]
    enc = (torch.randn(2, tlen, cfg.joint_attention_dim, generator=g) * 0.3).bfloat16().to(dev)
    mask = torch.ones(2, tlen, dtype=torch.long)
    mask[0, tlen // 3:] = 0
    mask = mask.to(dev)
    pooled = torch.randn(2, cfg.pooled_projection_dim, generator=g).to(dev)
    t = torch.tensor([700.0, 700.0], device=dev)
    model = B200FluxTransformer(FluxConfigB200(**kw), params, device=dev)
    ref = model(sample=[clips], timestep_ratio=t, encoder_hidden_states=enc, encoder_attention_mask=mask,
                pooled_projections=pooled)[0].float()
    seq = model.last_plan.seq
    if seq % lay.sp != 0:
        if rank == 0:
            print(f"[sp_check] {name}: S={seq} not divisible by sp={lay.sp}, skipped")
        continue
    for exchange, graph in (("nccl", False), ("peer", False), ("peer", True)):
        model.set_parallel_layout(lay, exchange=exchange)
        model.use_cuda_graph = graph
        worst = 0.0
        for rep in range(3 if graph else 1):            # capture, then replays
            out = model(sample=[clips], timestep_ratio=t, encoder_hidden_states=enc, encoder_attention_mask=mask,
                        pooled_projections=pooled)[0].float()
            torch.cuda.synchronize()
            worst = max(worst, (out - ref).abs().max().item())
        errs = [None] * world
        dist.all_gather_object(errs, worst)
        if rank == 0:
            print(f"[sp_check] {name}: world {world} = cfg {lay.cfg_ways} x sp {lay.sp} (heads {cfg.num_attention_heads} -> "
                  f"{SP.padded_heads(cfg.num_attention_heads, lay.sp)}), S={seq}, exchange={exchange}, graph={graph}: "
                  f"max|parallel - single| per rank = {['%.2e' % e for e in errs]}  |ref| mean {ref.abs().mean().item():.3f}", flush=True)
        assert worst < 2e-2, worst
    model.use_cuda_graph = False
# ---- SD3 MMDiT (24 heads; the reference runs it with sp 2 or 4)
from oracle import mmdit_oracle as MO
from pyramid_flow_b200.mmdit import B200MMDiT, MMDiTConfigB200
if 24 % lay.sp == 0:
    kw = dict(num_layers=3, pos_embed_max_size=96, sample_size=64)
    mcfg = MO.MMDiTConfig(**kw)
    params = MO.synthetic_mmdit_params(mcfg, seed=2)
    g = torch.Generator().manual_seed(6)
    clips = [torch.randn(s_, generator=g).bfloat16().to(dev) for s_ in [(2, 16, 2, 12, 20), (2, 16, 1, 24, 40), (2, 16, 1, 48, 80)]]
    enc = (torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().to(dev)
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[0, 50:] = 0
    mask = mask.to(dev)
    pooled = torch.randn(2, 2048, generator=g).to(dev)
    t = torch.tensor([500.0, 500.0], device=dev)
    model = B200MMDiT(MMDiTConfigB200(**{k_: v_ for k_, v_ in kw.items() if k_ != "sample_size"}), params, device=dev)
    call = dict(sample=[clips], timestep_ratio=t, encoder_hidden_states=enc, encoder_attention_mask=mask, pooled_projections=pooled)
    ref = model(**call)[0].float()
    if model.last_plan.seq % lay.sp == 0:
        model.set_parallel_layout(lay)
        out = model(**call)[0].float()
        torch.cuda.synchronize()
        err = (out - ref).abs().max().item()
        errs = [None] * world
        dist.all_gather_object(errs, err)
        if rank == 0:
            print(f"[sp_check] SD3 MMDiT (3 blocks): world {world} = cfg {lay.cfg_ways} x sp {lay.sp}, S={model.last_plan.seq}: "
                  f"max|parallel - single| per rank = {['%.2e' % e for e in errs]}  |ref| mean {ref.abs().mean().item():.3f}", flush=True)
        assert err < 2e-2, err
dist.destroy_process_group()
