"""Run ONE launch of a hot kernel at the bench shape (for `ncu --set full`): python tools/prof_one.py attn|gemm|ln"""
import sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch
from pyramid_flow_b200 import ops

which = sys.argv[1] if len(sys.argv) > 1 else "attn"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
dev = "cuda"
if which == "attn":
    B, H = 2, 30
    lens = [128 + 240] + [240] * 27 + [960, 3840, 3840]
    tim = torch.cat([torch.full((n,), float(i)) for i, n in enumerate(lens)]).int()[None].repeat(B, 1)
    S = tim.shape[1]
    seg = torch.ones(B, S, dtype=torch.int32)
    q = torch.randn(B, H, S, 64, device=dev).bfloat16()
    k = torch.randn(B, H, S, 64, device=dev).bfloat16()
    v = torch.randn(B, H, S, 64, device=dev).bfloat16()
    out = torch.zeros(B, S, H * 64, device=dev, dtype=torch.bfloat16)
    sched, pairs = ops.attn_build_schedule(seg, tim)
    ps = ops.attn_build_pair_schedule(sched, S, seg, tim).to(dev)
    sd, td, scd = seg.to(dev), tim.to(dev), sched.to(dev)
    variant = int(sys.argv[3], 0) if len(sys.argv) > 3 else 0        # pf_attn_desc.variant (every value runs the same kernel)
    for _ in range(reps):
        ops.attn_fwd(q, k, v, out, sd, td, scd, 0.125, variant=variant, pair_sched=ps)
elif which == "conv":
    # the widest full-resolution resnet conv of the VAE decode: 128 -> 128, 3x3x3, one 768x1280 frame chunk
    from pyramid_flow_b200.vae import B200CausalVAE, _Conv
    ci = co = 128
    t, h, w = 2, 768, 1280
    wt = (torch.randn(co, ci, 3, 3, 3) * (ci * 27) ** -0.5)
    cv = _Conv({"c.conv.weight": wt, "c.conv.bias": torch.zeros(co)}, "c", torch.device(dev))
    x = torch.randn(t + 2, h, w, ci, device=dev).bfloat16()
    out = torch.empty(t, h, w, co, device=dev, dtype=torch.bfloat16)
    holder = B200CausalVAE.__new__(B200CausalVAE)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(reps):
        if i == reps - 1:
            e0.record()
        B200CausalVAE._conv(holder, cv, x, t, h, w, out=out)
    e1.record()
    torch.cuda.synchronize()
    fl = 2.0 * 27 * ci * co * t * h * w
    print(f"conv 128->128 3x3x3 on {t}x{h}x{w}: {e0.elapsed_time(e1):.3f} ms, {fl / e0.elapsed_time(e1) / 1e9:.0f} TFLOP/s")
elif which == "gemm":
    m, n, k = 30976, 7680, 1920
    x = (torch.randn(m, k, device=dev) * 0.5).bfloat16()
    w = (torch.randn(n, k, device=dev) * 0.05).bfloat16()
    o = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
    for _ in range(reps):
        ops.gemm(x, w, None, 1, rows_per_batch=m, out=o)
torch.cuda.synchronize()
