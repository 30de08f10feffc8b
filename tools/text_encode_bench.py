"""Prompt encoding at full size: B200FluxTextEncoder (CLIP-L + T5-XXL) or, with --model mmdit, B200SD3TextEncoder
(CLIP-L + CLIP-G + T5-XXL), at B = 2 (one generate() call: prompt and negative prompt) and B = 64 (a caption batch of the
training-data recipe).

    python tools/text_encode_bench.py [--model flux|mmdit] [--batches 2 64] [--warmup 2] [--rounds 5] [--reference]
                                      [--json out.json]

The encoders have the released configurations (oracle.text_encoder_oracle CLIP_L / CLIP_G / T5_XXL) with seeded synthetic
weights at the init scales; the inputs are seeded token ids (CLIP: 77 tokens with BOS / EOS, T5: 128 tokens, every other
prompt padded after 37 tokens), so tokenisation is not timed.  Each batch size is warmed up, then timed `rounds` times (CUDA
events around one encode_ids call, median reported), with torch.cuda.max_memory_allocated over the timed rounds (weights
resident) and the host time until the call returned (launches are asynchronous: a host time close to the device time means
the GPU was waiting for the host).

--reference also builds the transformers models (CLIPTextModel / CLIPTextModelWithProjection / T5EncoderModel) in bf16 from
the same weights, on the same GPU, and times their eager forward on the same ids, alternating with ours round by round; it
prints the relative RMS difference of the two outputs.  The card's name, power limit and max SM clock are read with
nvidia-smi (a query only) in the same run.
"""
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from oracle import text_encoder_oracle as TO  # noqa: E402
from pyramid_flow_b200 import _lib  # noqa: E402
from pyramid_flow_b200.text_encoder import (B200CLIPText, B200FluxTextEncoder, B200SD3TextEncoder,  # noqa: E402
                                            B200T5Encoder)
from tools.vae_encode_bench import card  # noqa: E402


def seeded_ids(batch, seed=0):
    g = torch.Generator().manual_seed(seed)
    clip = torch.full((batch, 77), 49407, dtype=torch.long)
    clip[:, 0] = 49406
    clip[:, 1:40] = torch.randint(0, 49406, (batch, 39), generator=g)
    t5 = torch.randint(2, TO.T5_XXL.vocab_size, (batch, 128), generator=g)
    mask = torch.ones(batch, 128, dtype=torch.long)
    t5[::2, 127] = 1
    t5[1::2, 36] = 1
    t5[1::2, 37:] = 0
    mask[1::2, 37:] = 0
    return clip, t5, mask


def _hf(cls_fn, cfg, params, dev):
    """A transformers model of `cfg` in bf16 on `dev` holding `params`."""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)     # built in bf16 on the GPU: no fp32 copy of T5-XXL
    try:
        with torch.device(dev):
            m = cls_fn(cfg)
    finally:
        torch.set_default_dtype(prev)
    m = m.eval()
    sd = {k: v.to(torch.bfloat16) for k, v in params.items()}
    if "shared.weight" in sd:
        sd["encoder.embed_tokens.weight"] = sd["shared.weight"]
    m.load_state_dict(sd, strict=True)
    return m


def build(model, dev, reference):
    """(ours, reference forward or None)."""
    from transformers import CLIPTextModel, CLIPTextModelWithProjection, T5EncoderModel
    clip_cfgs = [TO.CLIP_L] if model == "flux" else [TO.CLIP_L_PROJ, TO.CLIP_G]
    clips, refs = [], []
    for i, cfg in enumerate(clip_cfgs):
        p = TO.synthetic_clip_params(cfg, seed=10 + i, device=dev)
        clips.append(B200CLIPText(cfg, p, dev))
        if reference:
            cls = CLIPTextModel if cfg.projection_dim is None else CLIPTextModelWithProjection
            refs.append(_hf(lambda c: cls(TO.hf_clip_config(c)), cfg, p, dev))
        del p
    p = TO.synthetic_t5_params(TO.T5_XXL, seed=20, device=dev)
    t5 = B200T5Encoder(TO.T5_XXL, p, dev)
    ref_t5 = _hf(lambda c: T5EncoderModel(TO.hf_t5_config(c)), TO.T5_XXL, p, dev) if reference else None
    del p
    torch.cuda.empty_cache()
    ours = B200FluxTextEncoder(None, None, clips[0], t5) if model == "flux" else \
        B200SD3TextEncoder(None, None, None, clips[0], clips[1], t5, tokenizer_max_length=77)

    def ours_fn(clip_ids, t5_ids, mask):
        if model == "flux":
            return ours.encode_ids(clip_ids, t5_ids, mask)
        return ours.encode_ids(clip_ids, clip_ids, t5_ids, mask)

    if not reference:
        return ours_fn, None

    @torch.no_grad()
    def ref_fn(clip_ids, t5_ids, mask):
        c, t, m = clip_ids.to(dev), t5_ids.to(dev), mask.to(dev)
        if model == "flux":
            pooled = refs[0](c).pooler_output
        else:
            pooled = torch.cat([r(c)[0] for r in refs], dim=-1)
        return ref_t5(t, attention_mask=m)[0], m, pooled

    return ours_fn, ref_fn


def time_once(fn, args):
    """(device ms between events around the call, host ms until the call returned, peak bytes, output).  A host time close
    to the device time means the GPU waited for launches."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    t0 = time.perf_counter()
    out = fn(*args)
    host_ms = (time.perf_counter() - t0) * 1e3
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), host_ms, torch.cuda.max_memory_allocated(), out


def rel_rms(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=("flux", "mmdit"), default="flux")
    ap.add_argument("--batches", type=int, nargs="+", default=[2, 64])
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    _lib.require_device()
    dev = torch.device("cuda:0")
    info = card()
    print(f"[text_encode_bench] {info['name']} | nvidia-smi name, power limit, max SM clock: {info['nvidia_smi']}")
    ours, ref = build(args.model, dev, args.reference)
    results = {"card": info, "model": args.model, "rows": []}
    for b in args.batches:
        ids = seeded_ids(b)
        impls = [("ours", ours)] + ([("reference", ref)] if ref else [])
        for _, fn in impls:
            for _ in range(args.warmup):
                fn(*ids)
        times = {n: [] for n, _ in impls}
        host = {n: [] for n, _ in impls}
        peaks = {n: 0 for n, _ in impls}
        outs = {}
        for _ in range(args.rounds):
            for n, fn in impls:       # alternating, round by round
                ms, host_ms, peak, out = time_once(fn, ids)
                times[n].append(ms)
                host[n].append(host_ms)
                peaks[n] = max(peaks[n], peak)
                outs[n] = out
        row = {"batch": b}
        for n, _ in impls:
            ms = statistics.median(times[n])
            row[n] = {"ms": ms, "host_ms": statistics.median(host[n]), "prompts_per_s": b / ms * 1e3,
                      "peak_gib": peaks[n] / 2 ** 30, "rounds_ms": times[n]}
        line = (f"[text_encode_bench] {args.model} B={b}: ours {row['ours']['ms']:.2f} ms ({row['ours']['prompts_per_s']:.0f} "
                f"prompts/s, peak {row['ours']['peak_gib']:.1f} GiB, host {row['ours']['host_ms']:.2f} ms)")
        if ref:
            r = row["reference"]
            o, w = outs["ours"], outs["reference"]
            row["embeds_rel_rms"], row["pooled_rel_rms"] = rel_rms(o[0], w[0]), rel_rms(o[2], w[2])
            line += (f" | transformers eager bf16 {r['ms']:.2f} ms ({r['prompts_per_s']:.0f} prompts/s, peak "
                     f"{r['peak_gib']:.1f} GiB, host {r['host_ms']:.2f} ms) | speed-up {r['ms'] / row['ours']['ms']:.2f}x | rel RMS diff embeds "
                     f"{row['embeds_rel_rms']:.2e} pooled {row['pooled_rel_rms']:.2e}")
        print(line, flush=True)
        results["rows"].append(row)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
