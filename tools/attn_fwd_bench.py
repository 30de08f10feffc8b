"""Per-launch time of the masked attention forward (pf_attn_fwd_masked) at the shape of the benchmarked DiT step, and an A/B
of library builds: every --lib is loaded into the same process, the builds are timed in alternation on the same inputs, and
their outputs are compared byte for byte with the first one's.

    python tools/attn_fwd_bench.py [--lib PATH ...] [--launches 20] [--rounds 6] [--warmup 3]

Shape: bench.py's step, B = 2, H = 30, S = 15488 (128 text tokens + the latent clips of bench.step_clip_shapes()), with the
seg / time ids and the tile schedule of dit.build_seq_plan and seeded normal bf16 q / k / v.  One round times --launches
back-to-back launches of each build between two CUDA events; the build order rotates from round to round.  Algorithmic
TFLOP/s counts 2 x 2 x 64 FLOP per allowed (q, kv) pair and head (Q.K^T and P.V).  One JSON line per build.  Without
--lib, the library of this tree is timed.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
from pyramid_flow_b200 import _lib  # noqa: E402
from pyramid_flow_b200.dit import build_seq_plan  # noqa: E402

HEADS, HEAD_DIM, TEXT = 30, 64, 128


def device_info(dev: torch.device) -> dict:
    info = {"device": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(dev.index or 0)], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = q
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = "unavailable"
    return info


def load_attention(path: Path):
    """pf_attn_fwd_masked of the library at `path` (each path is a separate copy of the library in this process)."""
    lib = C.CDLL(str(path))
    lib.pf_attn_fwd_masked.argtypes = [C.POINTER(_lib.AttnDesc), C.c_void_p]
    lib.pf_last_error.restype = C.c_char_p
    return lib


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", action="append", type=Path, default=None,
                    help="a libpf_b200.so build to time (repeatable; the first is the reference of the byte comparison)")
    ap.add_argument("--launches", type=int, default=20, help="launches per timed window")
    ap.add_argument("--rounds", type=int, default=6, help="timed windows per build, builds alternating")
    ap.add_argument("--warmup", type=int, default=3, help="untimed launches per build first")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_fwd_bench: needs an H100 (no CPU measurement path)")
    dev = torch.device("cuda:0")
    _lib.require_device()
    paths = args.lib or [_lib.LIB_PATH]
    libs = [load_attention(p.resolve()) for p in paths]

    b = 2
    plan = build_seq_plan(bench.step_clip_shapes(b), torch.ones(b, TEXT, dtype=torch.int64), (16, 24, 24), 2, dev)
    s = plan.seq
    g = torch.Generator(device=dev).manual_seed(0)
    q, k, v = (torch.randn(b, HEADS, s, HEAD_DIM, device=dev, dtype=torch.bfloat16, generator=g) for _ in range(3))
    outs = [torch.zeros(b, s, HEADS * HEAD_DIM, device=dev, dtype=torch.bfloat16) for _ in libs]
    descs = []
    for out in outs:
        d = _lib.AttnDesc()
        d.q, d.k, d.v, d.out, d.ldo = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), out.stride(1)
        d.batch, d.heads, d.seq, d.head_dim = b, HEADS, s, HEAD_DIM
        d.scale = HEAD_DIM ** -0.5
        d.seg, d.time, d.tile_sched, d.sched_stride = plan.seg.data_ptr(), plan.time.data_ptr(), plan.sched.data_ptr(), plan.sched.shape[-1]
        descs.append(d)

    def launch(i: int) -> None:
        rc = libs[i].pf_attn_fwd_masked(C.byref(descs[i]), C.c_void_p(_lib.stream_ptr()))
        if rc != 0:
            raise RuntimeError(f"{paths[i]}: pf_attn_fwd_masked failed ({rc}): {libs[i].pf_last_error().decode()}")

    # one launch each into a zeroed buffer: the bytes that are compared
    for i in range(len(libs)):
        launch(i)
    torch.cuda.synchronize()
    ref_bytes = outs[0].view(torch.int16)
    identical = [bool(torch.equal(o.view(torch.int16), ref_bytes)) for o in outs]
    max_abs = [float((o.float() - outs[0].float()).abs().max()) for o in outs]

    for i in range(len(libs)):
        for _ in range(args.warmup):
            launch(i)
    torch.cuda.synchronize()
    times = [[] for _ in libs]
    for r in range(args.rounds):
        for n in range(len(libs)):
            i = (r + n) % len(libs)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.launches):
                launch(i)
            e1.record()
            torch.cuda.synchronize()
            times[i].append(e0.elapsed_time(e1) / args.launches)

    flops = 4.0 * HEAD_DIM * HEADS * plan.allowed_pairs
    info = device_info(dev)
    for i, p in enumerate(paths):
        med = statistics.median(times[i])
        print(json.dumps({"lib": str(p), "batch": b, "heads": HEADS, "seq": s, "launches_per_window": args.launches,
                          "windows": args.rounds, "ms_per_launch_median": round(med, 4),
                          "ms_per_launch_min": round(min(times[i]), 4), "ms_per_launch_max": round(max(times[i]), 4),
                          "algorithmic_tflop_per_launch": round(flops / 1e12, 4),
                          "tflops_at_median": round(flops / (med * 1e-3) / 1e12, 1),
                          "output_bytes_equal_to_first": identical[i], "max_abs_diff_to_first": max_abs[i], **info}),
              flush=True)


if __name__ == "__main__":
    main()
