"""Training-path attention on the H100: the library's masked attention (forward + backward) against
F.scaled_dot_product_attention with the reference's dense bool mask; one whole call site (sources -> stage pack + RoPE ->
attention -> output split, forward + backward) against the reference's own glue + SDPA; and a reduced-depth reference DiT
training step with and without install_training_attention.  One JSON line per configuration.

    python tools/attn_train_bench.py [--iters 10] [--warmup 3] [--skip-dit] [--model flux|mmdit]

Attention shape: one stage of the autoregressive 768p training run (scripts/train_pyramid_flow.sh: batch 4, temporal
pyramid, temporal causal): 128 text tokens (T5 padding varies per sample), history frames at 1/4 and 1/2 of the 48 x 80 token
grid (1 x 12x20 + 2 x 24x40) and the current frame at full resolution (48x80): S = 6128, 24 heads of 64.  The call site is
that stage as a joint block sees it: bf16 q / k / v views of the Linear outputs (6000 video rows, 128 text rows), the temporal
RoPE table, the stage's plan or dense mask built beforehand (merge_input builds them once per step for every block).
The DiT step: the unmodified reference PyramidFluxTransformer (--model flux: miniFLUX width, 24 heads, 2 double + 4 single
blocks) or PyramidDiffusionMMDiT (--model mmdit: SD3 width, 24 heads, 4 joint blocks, the last context_pre_only, temporal
RoPE), staged under oracle/_ref, with gradient checkpointing, two pyramid stages of the same kind of layout, bf16 autocast.
Paired variants alternate in one process.  Times are CUDA-event medians; peak memory is torch's max_memory_allocated.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from pyramid_flow_b200 import _lib, training  # noqa: E402

DEV = torch.device("cuda:0")


def device_info() -> dict:
    info = {"device": torch.cuda.get_device_name(DEV)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = q
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = "unavailable"
    return info


def stage_layout(batch: int, text: int, frames):
    """seg / time int32 [batch, S]: text (sample b keeps text - 16 b tokens, the rest padded) then (n_frames, tokens) clips
    with consecutive time stamps."""
    segs, times = [], []
    for b in range(batch):
        valid = max(1, text - 16 * b)
        seg, time, stamp = [1] * valid + [0] * (text - valid), [0] * text, 0
        for t, n in frames:
            for f in range(t):
                seg += [1] * n
                time += [stamp + f] * n
            stamp += t
        segs.append(seg)
        times.append(time)
    return torch.tensor(segs, dtype=torch.int32), torch.tensor(times, dtype=torch.int32)


def timed(fn, iters: int, warmup: int):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times), min(times), max(times)


def peak_of(fn) -> int:
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def bench_attention(iters: int, warmup: int) -> list:
    batch, heads = 4, 24
    seg, time = stage_layout(batch, 128, [(1, 12 * 20), (2, 24 * 40), (1, 48 * 80)])
    s = seg.shape[1]
    g = torch.Generator(device=DEV).manual_seed(0)
    q, k, v, dout = (torch.randn(batch, heads, s, 64, device=DEV, dtype=torch.bfloat16, generator=g) for _ in range(4))
    segd, timed_ = seg.to(DEV), time.to(DEV)
    dout_rows = dout.transpose(1, 2).reshape(batch, s, heads * 64)

    def ours():
        qo, ko, vo = (t.detach().requires_grad_() for t in (q, k, v))
        training.masked_attention(qo, ko, vo, segd, timed_).backward(dout_rows)

    def sdpa():
        mask = (segd[:, :, None] == segd[:, None, :]) & (timed_[:, :, None] >= timed_[:, None, :])   # F:341-350
        qs, ks, vs = (t.detach().requires_grad_() for t in (q, k, v))
        F.scaled_dot_product_attention(qs, ks, vs, attn_mask=mask[:, None]).backward(dout)

    allowed = int(((seg[:, :, None] == seg[:, None, :]) & (time[:, :, None] >= time[:, None, :])).sum())
    flops = 4 * 64 * heads * allowed * 3.5      # fwd 2 GEMMs + bwd 5 GEMMs over the allowed pairs, 2 flop per MAC
    rows = []
    for name, fn in (("masked_attention", ours), ("sdpa_dense_mask", sdpa), ("masked_attention", ours), ("sdpa_dense_mask", sdpa)):
        med, lo, hi = timed(fn, iters, warmup)
        rows.append(dict(config="attention_fwd_bwd", impl=name, batch=batch, heads=heads, seq=s, ms_median=round(med, 3),
                         ms_min=round(lo, 3), ms_max=round(hi, 3), peak_mib=round(peak_of(fn) / 2**20, 1),
                         allowed_pair_fraction=round(allowed / (batch * s * s), 4),
                         tflops_on_allowed_pairs=round(flops / (med * 1e-3) / 1e12, 1)))
    return rows


def _reference():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        return None
    ref_shim.install()
    return ref_shim


def bench_call_site(iters: int, warmup: int) -> list:
    ref_shim = _reference()
    if ref_shim is None:
        return [dict(config="call_site_fwd_bwd", status="unavailable: the reference's sources are not staged (oracle/_ref)")]
    glue = __import__("pyramid_dit.mmdit_modules.modeling_mmdit_block",
                      fromlist=["VarlenSelfAttentionWithT5Mask"]).VarlenSelfAttentionWithT5Mask()
    batch, heads, text = 4, 24, 128
    seg, time = stage_layout(batch, text, [(1, 12 * 20), (2, 24 * 40), (1, 48 * 80)])
    s = seg.shape[1]
    rows_video = s - text
    g = torch.Generator(device=DEV).manual_seed(2)
    rnd = lambda *shape: torch.randn(*shape, device=DEV, dtype=torch.bfloat16, generator=g)
    video = [rnd(batch, rows_video, heads * 64) for _ in range(3)]        # to_q / to_k / to_v outputs
    enc = [rnd(batch, text, heads * 64) for _ in range(3)]                 # add_q / add_k / add_v outputs (one stage)
    ang = time.to(DEV).double()[..., None] / (10000 ** (torch.arange(0, 64, 2, device=DEV, dtype=torch.float64) / 64))
    freqs = torch.stack([ang.cos(), -ang.sin(), ang.sin(), ang.cos()], -1).view(batch, s, 32, 2, 2).float().unsqueeze(2)
    d_hid, d_enc = rnd(batch, rows_video, heads * 64), rnd(batch, text, heads * 64)
    segd, timed_ = seg.to(DEV), time.to(DEV)
    plan = training.plan_for(seg, time, DEV)
    dense = ((segd[:, :, None] == segd[:, None, :]) & (timed_[:, :, None] >= timed_[:, None, :]))[:, None]   # M:369-378

    def run(fn, mask):
        v = [t.detach().requires_grad_() for t in video]
        e = [t.detach().requires_grad_() for t in enc]
        hid, enc_out = fn(*(t.view(batch, -1, heads, 64) for t in v + e), heads, 0.125, hidden_length=[rows_video],
                          image_rotary_emb=[freqs], attention_mask=[mask])
        torch.autograd.backward([hid, enc_out], [d_hid, d_enc])

    ours = lambda: run(training._JointAttention(), plan)
    ref = lambda: run(glue, dense)
    rows = []
    for name, fn in (("library_pack_kernels", ours), ("reference_glue_sdpa", ref), ("library_pack_kernels", ours),
                     ("reference_glue_sdpa", ref)):
        med, lo, hi = timed(fn, iters, warmup)
        rows.append(dict(config="call_site_fwd_bwd", impl=name, batch=batch, heads=heads, seq=s, text=text,
                         ms_median=round(med, 3), ms_min=round(lo, 3), ms_max=round(hi, 3),
                         peak_mib=round(peak_of(fn) / 2**20, 1)))
    return rows


def _dit_model(ref_shim, kind: str):
    if kind == "flux":
        flux = __import__("pyramid_dit.flux_modules", fromlist=["PyramidFluxTransformer"]).PyramidFluxTransformer
        return flux(num_layers=2, num_single_layers=4, num_attention_heads=24, attention_head_dim=64, in_channels=64,
                    joint_attention_dim=4096, pooled_projection_dim=768, use_temporal_causal=True,
                    use_gradient_checkpointing=True, gradient_checkpointing_ratio=1.0), "2+4", 768
    mmdit = __import__("pyramid_dit.mmdit_modules", fromlist=["PyramidDiffusionMMDiT"]).PyramidDiffusionMMDiT
    return mmdit(num_layers=4, num_attention_heads=24, attention_head_dim=64, in_channels=16, caption_projection_dim=1536,
                 joint_attention_dim=4096, pooled_projection_dim=2048, pos_embed_type="sincos", temp_pos_embed_type="rope",
                 add_temp_pos_embed=True, use_flash_attn=False, use_temporal_causal=True, use_gradient_checkpointing=True,
                 gradient_checkpointing_ratio=1.0), "4 joint", 2048


def bench_dit(iters: int, warmup: int, kind: str) -> list:
    ref_shim = _reference()
    if ref_shim is None:
        return [dict(config="dit_train_step", status="unavailable: the reference's sources are not staged (oracle/_ref)")]
    model, blocks, pooled_dim = _dit_model(ref_shim, kind)
    ref_shim.reinit_all_parameters(model, seed=0, std=0.02)
    model = model.to(DEV).train()
    bs, text = 4, 128
    g = torch.Generator(device=DEV).manual_seed(1)
    rnd = lambda *shape: torch.randn(*shape, device=DEV, generator=g)
    # latents [b, 16, t, h, w] (tokens = t * h/2 * w/2); stage 0 current frame at 24 x 40 tokens, stage 1 at 48 x 80
    sample = [[rnd(bs, 16, 1, 24, 40), rnd(bs, 16, 1, 48, 80)],
              [rnd(bs, 16, 1, 24, 40), rnd(bs, 16, 2, 48, 80), rnd(bs, 16, 1, 96, 160)]]
    targets = [rnd(bs, 16, 1, 48, 80), rnd(bs, 16, 1, 96, 160)]
    enc, pooled = rnd(2 * bs, text, 4096), rnd(2 * bs, pooled_dim)
    mask = torch.ones(2 * bs, text, dtype=torch.long, device=DEV)
    for i in range(1, 2 * bs):
        mask[i, text - 9 * i:] = 0
    seq_per_stage = [text + sum(c.shape[2] * (c.shape[3] // 2) * (c.shape[4] // 2) for c in clips) for clips in sample]
    t = torch.tensor([900.0, 300.0] * bs, device=DEV)

    def step():
        model.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            preds = model(sample=sample, encoder_hidden_states=enc, encoder_attention_mask=mask, pooled_projections=pooled,
                          timestep_ratio=t)
            loss = sum(((p.float() - y) ** 2).mean() for p, y in zip(preds, targets))
        loss.backward()

    rows = []
    for installed in (False, True, False, True):
        if installed:
            training.install_training_attention(model)
        med, lo, hi = timed(step, iters, warmup)
        rows.append(dict(config="dit_train_step", model=kind, impl="installed" if installed else "reference_sdpa", blocks=blocks,
                         batch=bs, seq_per_stage=seq_per_stage,
                         ms_median=round(med, 2), ms_min=round(lo, 2), ms_max=round(hi, 2),
                         peak_mib=round(peak_of(step) / 2**20, 1)))
        training.uninstall_training_attention(model)
    return rows


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-dit", action="store_true")
    ap.add_argument("--skip-call-site", action="store_true")
    ap.add_argument("--model", choices=("flux", "mmdit"), default="flux", help="the reference DiT of the training-step leg")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_train_bench: needs an H100 (no CPU measurement path)")
    _lib.require_device()
    info = device_info()
    rows = bench_attention(args.iters, args.warmup)
    if not args.skip_call_site:
        rows += bench_call_site(args.iters, args.warmup)
    if not args.skip_dit:
        rows += bench_dit(args.iters, args.warmup, args.model)
    for r in rows:
        print(json.dumps({**r, **info}), flush=True)


if __name__ == "__main__":
    main()
