"""The DiT step with bf16 GEMMs and with gemm_precision="fp8", built from the same synthetic weights and timed in one process.

    python tools/fp8_step_bench.py [--model flux|mmdit] [--steps 10] [--warmup 3] [--rounds 3] [--json out.json]

--model flux (default): bench.py's miniFLUX workload (B=2, S=15488, 8 double + 16 single blocks).
--model mmdit: bench.py --model mmdit's SD3 MMDiT workload (B=2, S=11888, 24 joint blocks, D=1536).

Each round times `steps` graph-replayed steps of the bf16 model, then of the fp8 model (CUDA events, after `warmup` steps),
so that the two alternate `rounds` times.  Then one extra step per precision runs host-launched, and the velocity of each
precision is compared with the other's (fp32 stores).  For miniFLUX that step also runs the model's kernel-family timer
(CUDA events around every launch: the quantise passes are "quantize_fp8").  The card's name, power limit and max SM clock
are read with nvidia-smi (a query only).
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

from bench import random_flux_state_dict, random_mmdit_state_dict, step_clip_shapes  # noqa: E402
from pyramid_flow_b200 import _lib  # noqa: E402
from pyramid_flow_b200.dit import B200FluxTransformer  # noqa: E402
from pyramid_flow_b200.mmdit import B200MMDiT, MMDiTConfigB200  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": out or "unavailable"}


def flux_models(dev):
    cfg, sd = random_flux_state_dict({}, dev, seed=0)
    models = {p: B200FluxTransformer(cfg, sd, device=dev, gemm_precision=p) for p in ("bf16", "fp8")}
    g = torch.Generator().manual_seed(100)
    call = dict(sample=[[torch.randn(s, generator=g).bfloat16().to(dev) for s in step_clip_shapes(2)]],
                timestep_ratio=torch.tensor([3.0, 3.0]).bfloat16().to(dev),
                encoder_hidden_states=(torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().to(dev),
                encoder_attention_mask=torch.ones(2, 128, dtype=torch.int64, device=dev),
                pooled_projections=torch.randn(2, 768, generator=g).bfloat16().to(dev))
    return models, call


def mmdit_models(dev):
    """bench.run_mmdit's model and inputs: S = 128 + 13x240 + 960 + 2x3840 = 11888."""
    cfg = MMDiTConfigB200()
    sd = random_mmdit_state_dict(cfg, dev)
    models = {p: B200MMDiT(cfg, sd, device=dev, gemm_precision=p) for p in ("bf16", "fp8")}
    g = torch.Generator().manual_seed(100)
    shapes = [(2, 16, 13, 24, 40), (2, 16, 1, 48, 80), (2, 16, 1, 96, 160), (2, 16, 1, 96, 160)]
    call = dict(sample=[[torch.randn(s, generator=g).bfloat16().to(dev) for s in shapes]],
                encoder_hidden_states=(torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().to(dev),
                encoder_attention_mask=torch.ones(2, 128, dtype=torch.int64, device=dev),
                pooled_projections=torch.randn(2, 2048, generator=g).bfloat16().to(dev),
                timestep_ratio=torch.tensor([3.0, 3.0]).bfloat16().to(dev))
    return models, call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="flux", choices=["flux", "mmdit"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    _lib.require_device()
    dev = torch.device("cuda:0")
    info = card()
    print(f"[fp8_step_bench] {info['name']} | nvidia-smi name, power limit, max SM clock: {info['nvidia_smi']}")

    models, call = (flux_models if args.model == "flux" else mmdit_models)(dev)
    torch.cuda.empty_cache()

    def timed(model):
        for _ in range(args.warmup):
            model(**call)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            model(**call)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    ms = {p: [] for p in models}
    for m in models.values():
        m.use_cuda_graph = True
    for r in range(args.rounds):
        for p, m in models.items():
            ms[p].append(timed(m))
        print(f"[fp8_step_bench] round {r}: bf16 {ms['bf16'][-1]:.2f} ms/step, fp8 {ms['fp8'][-1]:.2f} ms/step")
    med = {p: statistics.median(v) for p, v in ms.items()}
    print(f"[fp8_step_bench] median over {args.rounds} rounds of {args.steps} graph-replayed steps: bf16 {med['bf16']:.2f} ms, "
          f"fp8 {med['fp8']:.2f} ms ({med['bf16'] / med['fp8']:.3f}x)")

    breakdown, vel = {}, {}
    for p, m in models.items():
        m.use_cuda_graph = False
        if args.model == "mmdit":   # fp32 clips holding the same bf16 values: the same step with an fp32 velocity store
            vel[p] = m(**dict(call, sample=[[c.float() for c in call["sample"][0]]]))[0]
            continue
        m.output_fp32 = True
        m.timer.enabled = True
        m.timer.events = []
        m.attn_events = []
        vel[p] = m(**call)[0].float()
        torch.cuda.synchronize()
        bd = m.timer.totals_ms()
        bd["attention"] = sum(a.elapsed_time(b) for a, b in m.attn_events)
        m.timer.enabled = False
        m.attn_events = None
        breakdown[p] = {k: round(v, 3) for k, v in sorted(bd.items())}
        print(f"[fp8_step_bench] {p} per-family breakdown of one host-launched step (ms): {breakdown[p]}")
    d = vel["fp8"] - vel["bf16"]
    err = dict(max_abs=d.abs().max().item(), rel_rms=(d.pow(2).mean().sqrt() / vel["bf16"].pow(2).mean().sqrt()).item(),
               cosine=torch.nn.functional.cosine_similarity(vel["fp8"].flatten().double(), vel["bf16"].flatten().double(),
                                                            dim=0).item())
    print(f"[fp8_step_bench] fp8 velocity vs bf16 velocity (fp32 stores): {err}")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(dict(card=info, model=args.model, ms_per_step=ms, median_ms=med,
                                                   breakdown_ms=breakdown, fp8_vs_bf16=err), indent=1))


if __name__ == "__main__":
    main()
