"""Time every GEMM family of one DiT step at the step's exact shapes and epilogues (B=2, S=15488 = 128 text + 15360 video
tokens, 30 heads x 64, FF 4x), through pf_gemm_bf16, or with --fp8 through pf_gemm_fp8 on e4m3 operands (the same rows; the
rate is printed next to the H100 SXM data-sheet bound, 989 TFLOP/s dense bf16 and 1,979 dense fp8, a bound that is not reached).

    python tools/gemm_bench.py [--fp8] [--iters 30] [--warmup 5] [--json out.json]

Each row is timed with CUDA events around `iters` back-to-back launches after `warmup` launches of the same shape; the rate is
2*M*N*K over the mean launch time.  Operands are re-read every launch, and every row's working set (A + W + output) is larger
than H100's 50 MB L2 except the 128-row text ranges, so what is timed is the kernel streaming from HBM as in the step.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from pyramid_flow_b200 import _lib, ops  # noqa: E402
from pyramid_flow_b200._lib import PF_EPI_GATE_RESID, PF_EPI_GELU_BF16, PF_EPI_QKV_ROPE  # noqa: E402

B, TXT, VID, H, HD = 2, 128, 15360, 30, 64
S = TXT + VID
D = H * HD
L2_BYTES = 50 * 2**20

# (family, row_begin, row_count, n, k, epilogue, launches per step)
ROWS = [
    ("gemm_qkv double video", TXT, VID, 3 * D, D, PF_EPI_QKV_ROPE, 8),
    ("gemm_qkv double text", 0, TXT, 3 * D, D, PF_EPI_QKV_ROPE, 8),
    ("gemm_qkv single", 0, S, 3 * D, D, PF_EPI_QKV_ROPE, 16),
    ("gemm_ff1_gelu video", TXT, VID, 4 * D, D, PF_EPI_GELU_BF16, 8),
    ("gemm_ff1_gelu text", 0, TXT, 4 * D, D, PF_EPI_GELU_BF16, 8),
    ("gemm_single_mlp_gelu", 0, S, 4 * D, D, PF_EPI_GELU_BF16, 16),
    ("gemm_attn_out video", TXT, VID, D, D, PF_EPI_GATE_RESID, 8),
    ("gemm_attn_out text", 0, TXT, D, D, PF_EPI_GATE_RESID, 8),
    ("gemm_ff2 video", TXT, VID, D, 4 * D, PF_EPI_GATE_RESID, 8),
    ("gemm_ff2 text", 0, TXT, D, 4 * D, PF_EPI_GATE_RESID, 8),
    ("gemm_single_out", 0, S, D, 5 * D, PF_EPI_GATE_RESID, 16),
]


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": out or "unavailable"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kernel-variant", type=int, default=0, help="pf_gemm_desc.kernel_variant (0 = automatic choice)")
    ap.add_argument("--fp8", action="store_true", help="pf_gemm_fp8 on e4m3 operands with per-row / per-channel scales")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    bound = 1979.0 if args.fp8 else 989.0
    _lib.require_device()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    xn = (torch.randn(B, S, 5 * D, device=dev, generator=g) * 0.5).bfloat16()      # widest A (single_out's K = 5*D)
    h = torch.randn(B, S, D, device=dev, generator=g)
    out = torch.empty(B, S, 4 * D, device=dev, dtype=torch.bfloat16)
    q, k, v = (torch.empty(B, H, S, HD, device=dev, dtype=torch.bfloat16) for _ in range(3))
    ang = torch.randn(S, HD // 2, device=dev, generator=g)
    rope = torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous()
    nq = 1 + 0.1 * torch.randn(HD, device=dev, generator=g)
    nk = 1 + 0.1 * torch.randn(HD, device=dev, generator=g)
    gate = torch.randn(B, D, device=dev, generator=g) * 0.01
    if args.fp8:
        xn8 = torch.empty(B, S, 5 * D, device=dev, dtype=torch.float8_e4m3fn)
        sa = torch.empty(B, S, device=dev)
        ops.quantize_rows_fp8(xn, xn8, sa, batches=B, rows_per_batch=S)
    info = card()
    print(f"[gemm_bench] {info['name']} | nvidia-smi name, power limit, max SM clock: {info['nvidia_smi']}")
    print(f"[gemm_bench] CUDA events over {args.iters} back-to-back launches after {args.warmup} warm-up launches; "
          f"L2 = 50 MB, working set (A + W + out) per row below")
    rows, total_ms, total_flop = [], 0.0, 0.0
    for name, r0, rc, n, kk, epi, per_step in ROWS:
        a = xn[:, :, :kk]
        w = (torch.randn(n, kk, device=dev, generator=g) * 0.02).bfloat16()
        if args.fp8:
            w8, sw = (t.to(dev) for t in ops.quantize_weight_fp8(w.cpu()))
            a8 = xn8[:, :, :kk]
        bias = torch.randn(n, device=dev, generator=g) * 0.1
        if epi == PF_EPI_QKV_ROPE:
            kw = dict(q_out=q, k_out=k, v_out=v, rope=rope, q_norm_w=nq, k_norm_w=nk, heads=H, head_dim=HD, seq_len=S)
            out_bytes = B * rc * n * 2
        elif epi == PF_EPI_GELU_BF16:
            kw = dict(out=out[:, :, :n], ldo=4 * D)
            out_bytes = B * rc * n * 2
        else:
            kw = dict(out=h, ldo=D, gate=gate, gate_batch_stride=D)
            out_bytes = 2 * B * rc * n * 4

        def launch():
            if args.fp8:
                ops.gemm_fp8(a8, sa, w8, sw, bias, epi, batches=B, rows_per_batch=S, row_begin=r0, row_count=rc, **kw)
            else:
                ops.gemm(a, w, bias, epi, batches=B, rows_per_batch=S, row_begin=r0, row_count=rc,
                         kernel_variant=args.kernel_variant, **kw)
        for _ in range(args.warmup):
            launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.iters):
            launch()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        flop = 2.0 * B * rc * n * kk
        esz = 1 if args.fp8 else 2
        ws = B * rc * kk * esz + n * kk * esz + out_bytes
        tf = flop / (ms * 1e-3) / 1e12
        total_ms += ms * per_step
        total_flop += flop * per_step
        rows.append(dict(family=name, m=B * rc, n=n, k=kk, ms=round(ms, 4), tflops=round(tf, 1), per_step=per_step,
                         working_set_mb=round(ws / 2**20, 1)))
        print(f"  {name:24s} M={B * rc:6d} N={n:5d} K={kk:5d}  {ms * 1e3:9.1f} us  {tf:6.1f} TFLOP/s "
              f"(data-sheet bound {bound:.0f})  "
              f"x{per_step:2d}/step  working set {ws / 2**20:7.1f} MB {'> L2' if ws > L2_BYTES else '< L2'}")
    print(f"[gemm_bench] per-step GEMM total (rows above x launches/step): {total_ms:.2f} ms, "
          f"{total_flop / (total_ms * 1e-3) / 1e12:.1f} TFLOP/s")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(dict(card=info, fp8=args.fp8, rows=rows, step_total_ms=round(total_ms, 3)),
                                              indent=1))


if __name__ == "__main__":
    main()
