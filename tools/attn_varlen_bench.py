"""The flash-path (varlen) training attention on the H100, forward + backward, at the shapes of the no-AR recipe
(scripts/train_pyramid_flow_without_ar.sh, batch 4, 128 T5 tokens with padding that varies per sample):

  * t2i_768p: 768p images (1280 x 768 -> 160 x 96 latent -> 80 x 48 tokens after the 2 x 2 patch); the three pyramid stages
    (stages=[1, 2, 4] of PyramidDiTForVideoGeneration) at 1/4, 1/2 and full resolution: 240, 960 and 3840 video tokens.
  * t2v_384p: a full-sequence 384p clip of 16 latent frames (--max_frames 16, 5 s; 640 x 384 -> 40 x 24 tokens a frame),
    each stage the whole clip: 16 x 60, 16 x 240 and 16 x 960 video tokens.

Legs, one JSON line each, paired variants alternating in one process:
  * varlen_attention against flash_attn_varlen_func on the packed sequences of one call site ("not available" when
    flash_attn does not import);
  * one double-block call site (q / k / v views of the Linear outputs and the RoPE tables -> outputs) through the library
    against the reference's own glue (VarlenFlashSelfAttentionWithT5Mask) with FA2 and with a torch stand-in (per-sequence SDPA);
  * a reduced-depth reference miniFLUX training step (miniFLUX width, 24 heads, 2 double + 4 single blocks, gradient
    checkpointing, bf16 parameters and autocast, t2i_768p) with and without install_varlen_training_attention.

    python tools/attn_varlen_bench.py [--iters 10] [--warmup 3] [--skip-dit]

Times are CUDA-event medians; peak memory is torch's max_memory_allocated above what was allocated before the call.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from pyramid_flow_b200 import _lib, training  # noqa: E402
from tools.attn_train_bench import DEV, device_info, peak_of, timed  # noqa: E402

BATCH, HEADS, TEXT = 4, 24, 128
SHAPES = {"t2i_768p": [240, 960, 3840], "t2v_384p": [16 * 60, 16 * 240, 16 * 960]}


def _flash():
    try:
        from flash_attn.flash_attn_interface import flash_attn_varlen_func
        return flash_attn_varlen_func
    except ImportError:
        return None


# torch stand-ins for the flash_attn helpers the reference's glue calls
def index_first_axis(x, indices):
    return x[indices]


def pad_input(x, indices, batch, seqlen):
    out = torch.zeros(batch * seqlen, *x.shape[1:], dtype=x.dtype, device=x.device)
    out[indices] = x
    return out.view(batch, seqlen, *x.shape[1:])


def varlen_standin(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dropout_p=0.0, causal=False,
                   softmax_scale=None):
    cu = cu_seqlens_q.tolist()
    return torch.cat([F.scaled_dot_product_attention(*(t[a:b].transpose(0, 1)[None] for t in (q, k, v)),
                                                     scale=softmax_scale)[0].transpose(0, 1) for a, b in zip(cu[:-1], cu[1:])])


def _mask(n_stages):
    """Encoder mask [B * n_stages, 128]: row r keeps 128 - 9 r tokens (at least 1)."""
    mask = torch.zeros(BATCH * n_stages, TEXT, dtype=torch.long, device=DEV)
    for r in range(BATCH * n_stages):
        mask[r, :max(1, TEXT - 9 * r)] = 1
    return mask


def _stages(mask, hidden_length):
    """merge_input's flash branch (F:295-317)."""
    n, out = len(hidden_length), []
    for i, length in enumerate(hidden_length):
        m = torch.cat([mask[i::n], torch.ones(BATCH, length, dtype=mask.dtype, device=DEV)], dim=1)
        out.append({"indices": torch.nonzero(m.flatten()).flatten(), "seqlens_in_batch": m.sum(-1, dtype=torch.int32)})
    return out


def _rope(b, seq, g):
    pos = torch.randint(0, 64, (b, seq), device=DEV, generator=g).double()
    ang = pos[..., None] / (10000 ** (torch.arange(0, 64, 2, device=DEV, dtype=torch.float64) / 64))
    return torch.stack([ang.cos(), -ang.sin(), ang.sin(), ang.cos()], -1).view(b, seq, 32, 2, 2).float().unsqueeze(2)


def _row(config, shape, impl, fn, iters, warmup, **extra):
    med, lo, hi = timed(fn, iters, warmup)
    return dict(config=config, shape=shape, impl=impl, ms_median=round(med, 3), ms_min=round(lo, 3), ms_max=round(hi, 3),
                peak_mib=round(peak_of(fn) / 2**20, 1), **extra)


def bench_attention(shape, iters, warmup) -> list:
    hidden_length = SHAPES[shape]
    stages = _stages(_mask(3), hidden_length)
    seqlens = torch.cat([s["seqlens_in_batch"] for s in stages])
    cu = F.pad(torch.cumsum(seqlens, 0, dtype=torch.int32), (1, 0))
    total, mx = int(cu[-1]), int(seqlens.max())
    g = torch.Generator(device=DEV).manual_seed(0)
    q, k, v, dout = (torch.randn(total, HEADS, 64, device=DEV, dtype=torch.bfloat16, generator=g) for _ in range(4))
    fa = _flash()

    def run(fn):
        def go():
            qs, ks, vs = (t.detach().requires_grad_() for t in (q, k, v))
            fn(qs, ks, vs).backward(dout)
        return go

    ours = run(lambda a, b, c: training.varlen_attention(a, b, c, cu, softmax_scale=0.125))
    extra = dict(batch=BATCH, heads=HEADS, total_rows=total, sequences=int(seqlens.numel()), max_seqlen=mx)
    rows = []
    for _ in range(2):
        rows.append(_row("varlen_attention_fwd_bwd", shape, "library", ours, iters, warmup, **extra))
        if fa is None:
            rows.append(dict(config="varlen_attention_fwd_bwd", shape=shape, impl="flash_attn", status="not available"))
        else:
            rows.append(_row("varlen_attention_fwd_bwd", shape, "flash_attn",
                             run(lambda a, b, c: fa(a, b, c, cu, cu, mx, mx, softmax_scale=0.125)), iters, warmup, **extra))
    return rows


def _reference():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        return None
    ref_shim.install()
    return ref_shim


def bench_call_site(shape, iters, warmup) -> list:
    if _reference() is None:
        return [dict(config="call_site_fwd_bwd", shape=shape, status="unavailable: the reference's sources are not staged")]
    block = __import__("pyramid_dit.flux_modules.modeling_flux_block", fromlist=["VarlenFlashSelfAttentionWithT5Mask"])
    hidden_length = SHAPES[shape]
    n, s = len(hidden_length), sum(hidden_length)
    mask = _mask(n)
    stages = _stages(mask, hidden_length)
    plan = training.varlen_plan([st["indices"] for st in stages], [st["seqlens_in_batch"] for st in stages], BATCH,
                                [TEXT + L for L in hidden_length])
    g = torch.Generator(device=DEV).manual_seed(2)
    rnd = lambda *sh: torch.randn(*sh, device=DEV, dtype=torch.bfloat16, generator=g)
    video = [rnd(BATCH, s, HEADS * 64) for _ in range(3)]
    enc = [rnd(BATCH * n, TEXT, HEADS * 64) for _ in range(3)]
    freqs = [_rope(BATCH, TEXT + L, g) for L in hidden_length]
    d_hid, d_enc = rnd(BATCH, s, HEADS * 64), rnd(BATCH * n, TEXT, HEADS * 64)

    def run(fn, arg):
        def go():
            v = [t.detach().requires_grad_() for t in video]
            e = [t.detach().requires_grad_() for t in enc]
            hid, enc_out = fn(*(t.view(t.shape[0], -1, HEADS, 64) for t in v + e), HEADS, 0.125, hidden_length, freqs, arg)
            torch.autograd.backward([hid, enc_out], [d_hid, d_enc])
        return go

    fa = _flash()
    glue = block.VarlenFlashSelfAttentionWithT5Mask()
    saved = {k: getattr(block, k, None) for k in ("flash_attn_varlen_func", "index_first_axis", "pad_input")}

    def with_impl(impl, go):
        def wrapped():
            if impl == "standin":
                block.flash_attn_varlen_func, block.index_first_axis, block.pad_input = varlen_standin, index_first_axis, pad_input
            try:
                go()
            finally:
                for k, val in saved.items():
                    setattr(block, k, val)
        return wrapped

    extra = dict(batch=BATCH, heads=HEADS, text=TEXT, video_rows=s, packed_rows=plan.total)
    rows = []
    for _ in range(2):
        rows.append(_row("call_site_fwd_bwd", shape, "library", run(training._VarlenJointAttention(), plan), iters, warmup, **extra))
        if fa is None or saved["pad_input"] is None:
            rows.append(dict(config="call_site_fwd_bwd", shape=shape, impl="reference_glue_fa2", status="not available"))
        else:
            rows.append(_row("call_site_fwd_bwd", shape, "reference_glue_fa2", run(glue, stages), iters, warmup, **extra))
        rows.append(_row("call_site_fwd_bwd", shape, "reference_glue_standin", with_impl("standin", run(glue, stages)), iters,
                         warmup, **extra))
    return rows


def bench_dit(iters, warmup) -> list:
    ref_shim = _reference()
    if ref_shim is None:
        return [dict(config="dit_train_step", status="unavailable: the reference's sources are not staged")]
    flux = __import__("pyramid_dit.flux_modules", fromlist=["PyramidFluxTransformer"]).PyramidFluxTransformer
    block = sys.modules["pyramid_dit.flux_modules.modeling_flux_block"]
    model = flux(num_layers=2, num_single_layers=4, num_attention_heads=HEADS, attention_head_dim=64, in_channels=64,
                 joint_attention_dim=4096, pooled_projection_dim=768, use_flash_attn=True, use_gradient_checkpointing=True,
                 gradient_checkpointing_ratio=1.0)
    ref_shim.reinit_all_parameters(model, seed=0, std=0.02)
    model = model.to(DEV, torch.bfloat16).train()        # --model_dtype bf16, as the recipe trains
    g = torch.Generator(device=DEV).manual_seed(1)
    rnd = lambda *sh: torch.randn(*sh, device=DEV, generator=g).to(torch.bfloat16)
    # t2i_768p latents [b, 16, 1, h, w] at 1/4, 1/2 and full resolution (tokens = h/2 * w/2)
    sample = [[rnd(BATCH, 16, 1, 24, 40)], [rnd(BATCH, 16, 1, 48, 80)], [rnd(BATCH, 16, 1, 96, 160)]]
    targets = [c[0].clone() for c in sample]
    enc, pooled, mask = rnd(3 * BATCH, TEXT, 4096), rnd(3 * BATCH, 768), _mask(3)
    t = torch.tensor([900.0, 500.0, 100.0] * BATCH, device=DEV, dtype=torch.bfloat16)

    def step():
        model.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            preds = model(sample=sample, encoder_hidden_states=enc, encoder_attention_mask=mask, pooled_projections=pooled,
                          timestep_ratio=t)
            loss = sum(((p.float() - y) ** 2).mean() for p, y in zip(preds, targets))
        loss.backward()

    fa = _flash()
    saved = {k: getattr(block, k, None) for k in ("flash_attn_varlen_func", "index_first_axis", "pad_input")}
    ref_impl = "reference_fa2" if fa is not None and saved["pad_input"] is not None else "reference_standin"
    extra = dict(blocks="2+4", batch=BATCH, seq_per_stage=[TEXT + 12 * 20, TEXT + 24 * 40, TEXT + 48 * 80])
    rows = []
    try:
        if ref_impl == "reference_standin":
            block.flash_attn_varlen_func, block.index_first_axis, block.pad_input = varlen_standin, index_first_axis, pad_input
        for installed in (False, True, False, True):
            if installed:
                training.install_varlen_training_attention(model)
            rows.append(_row("dit_train_step", "t2i_768p", "installed" if installed else ref_impl, step, iters, warmup, **extra))
            training.uninstall_training_attention(model)
    finally:
        for k, val in saved.items():
            setattr(block, k, val)
    return rows


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-dit", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_varlen_bench: needs an H100 (no CPU measurement path)")
    _lib.require_device()
    info = device_info()
    legs = [(fn, shape) for shape in SHAPES for fn in (bench_attention, bench_call_site)]
    if not args.skip_dit:
        legs.append((lambda iters, warmup: bench_dit(iters, warmup), None))
    for fn, shape in legs:
        for r in (fn(shape, args.iters, args.warmup) if shape is not None else fn(args.iters, args.warmup)):
            print(json.dumps({**r, **info}), flush=True)


if __name__ == "__main__":
    main()
