"""Training convolutions of the causal video VAE on the H100: per conv family, the library's forward / data gradient /
weight gradient against torch's bf16 autocast conv3d + autograd (cuDNN), the pack passes on their own lines, and a
full-size reference CausalVideoVAE training step with and without install_training_convs (and with install_training_norms
on top).  One JSON line per measurement.

    python tools/vae_train_bench.py [--iters 10] [--warmup 3] [--rounds 3] [--skip-step] [--skip-norms] [--skip-profile]

Shapes: the stage-1 run of scripts/train_causal_video_vae.sh -- batch 2, 17 frames, 256 x 256, the full-size VAE's
channels (128 / 256 / 512 / 512); each conv family is timed at the level of the encoder where it runs.  TFLOP/s are
algorithmic: 2 * output voxels * Cout * Cin * taps for each of forward, data and weight gradient (the data gradient of a
strided conv runs over the zero-inserted grid, 4x resp. 2x that work, which the rate does not count).  cuDNN's weight
gradient is timed without its bias gradient, which the library computes in its dy pack (the pack_dy_db line).  Lines
"<pass>:<kernel>" give the device time of each kernel inside the library's wgrad and dy-pack calls (torch.profiler, after
the timed runs): the GEMM and the split reduce, the pack and the two bias-gradient reduce passes.  The training step
is encode -> posterior.sample() -> decode -> L1 + KL -> backward under bf16 autocast on synthetic weights, for the video
clip and for a batch of 8 images (T = 1); LPIPS needs a checkpoint and the discriminator starts at step 250000, so the
step leaves both out.  Paired variants alternate in one process; times are CUDA-event medians; peak memory is torch's
max_memory_allocated.

Norm families: hooks record the shape, layout form and dtype of every CausalGroupNorm input, and the layout its output's
gradient arrives in, during one step of the video clip with the convolutions and the norms installed; for each distinct
family (the site names are listed) the library's causal_group_norm (SiLU fused, bf16 output, as install_training_norms
runs it) is timed forward and forward + backward, x and dy in those layouts (a gradient copied into x's form is part of
the time), against the reference module + nn.SiLU under bf16 autocast, with the rel. RMS of the two outputs (torch's fp32
output rounded to bf16) and of the input gradients against each other.  The
step reports how many norm inputs / gradients causal_group_norm had to copy into a layout its kernels read.  A separate
torch.profiler pass of the convs-only and the convs + norms steps gives the device time of torch's GroupNorm / SiLU ops
(forward and backward) and of the conv pack kernel.

LPIPS (--skip-lpips to leave it out): the recipe's generator step with the real loss -- LPIPSWithDiscriminator at the
stage-1 weights (pixel 10, perceptual 1, KL 1e-12, disc_start 250000, so the discriminator does not run) with a synthetic
LPIPS checkpoint from a fixed seed, in training mode (LPIPS's dropout live) -- for torch, convs + norms and convs + norms +
LPIPS, alternating, with peak memory.  LPIPS alone at the clip shape (34 + 34 frames of 256^2: B = 2 x 17 frames per
branch) and the image shape (8 + 8): the library's lpips against the reference module under bf16 autocast, forward and
forward + backward (gradient to the reconstruction only, as in the loss), with peak memory and algorithmic TFLOP/s
(2 * H * W * Cin * Cout * 9 per conv and image: forward over both branches, data gradient over one; the first conv's
3 input channels are counted as 3, not as the 64 the kernel computes).  A separate line times the first conv alone
(3 -> 64 channels padded to 64 -> 64) and gives its padded and real FLOP counts; a profiler pass gives each kernel family's
device time: VGG convs (forward pass), data-gradient convs (the rest of the conv kernel's time in forward + backward),
pool, head, tap backward and the input pack.
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

from pyramid_flow_b200 import _lib, ops, vae_training as VT  # noqa: E402

DEV = torch.device("cuda:0")

# name, cin, cout, k, stride, (t, h, w) of the conv's INPUT
FAMILIES = [
    ("k3_c128", 128, 128, 3, (1, 1, 1), (17, 256, 256)),
    ("k3_c256", 256, 256, 3, (1, 1, 1), (9, 128, 128)),
    ("k3_c512", 512, 512, 3, (1, 1, 1), (5, 64, 64)),
    ("down_s122_c128", 128, 128, 3, (1, 2, 2), (17, 256, 256)),
    ("down_s211_c128", 128, 128, 3, (2, 1, 1), (17, 128, 128)),
    ("shortcut_k1_c128to256", 128, 256, 1, (1, 1, 1), (9, 128, 128)),
    ("up_x4_c512", 512, 2048, 3, (1, 1, 1), (3, 32, 32)),
    ("up_t2_c512", 512, 1024, 3, (1, 1, 1), (3, 64, 64)),
]


def device_info() -> dict:
    info = {"device": torch.cuda.get_device_name(DEV)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = q
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = "unavailable"
    return info


def timed(fn, iters: int, warmup: int) -> float:
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
    return statistics.median(times)


def rel_rms(a, ref) -> float:
    a, ref = a.float(), ref.float()
    return ((a - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt().clamp_min(1e-30)).item()


def bench_family(name, cin, cout, k, stride, thw, iters, warmup, batch=2) -> list:
    g = torch.Generator(device=DEV).manual_seed(0)
    t, h, w = thw
    x = torch.randn(batch, cin, t, h, w, device=DEV, generator=g, dtype=torch.bfloat16)
    wt = torch.randn(cout, cin, k, k, k, device=DEV, generator=g) * (1.0 / (cin * k ** 3) ** 0.5)
    bias = torch.randn(cout, device=DEV, generator=g) * 0.1
    to, ho, wo = VT._out_dims(x.shape, stride)
    dy = torch.randn(batch, cout, to, ho, wo, device=DEV, generator=g, dtype=torch.bfloat16)
    flops = 2.0 * batch * to * ho * wo * cout * cin * k ** 3
    kt = k
    cin_p, cout_p = VT._pad64(cin), VT._pad64(cout)

    # ---- library: the passes of causal_conv3d's forward / backward, one at a time
    t_in = (to - 1) * stride[0] + kt
    xp = torch.empty(batch, t_in, h, w, cin_p, device=DEV, dtype=torch.bfloat16)
    xs = x[:, :, :t_in - (kt - 1)]
    xs32 = xs.float()
    wf, wb = VT.forward_filter(wt, cout_p, cin_p), VT.dgrad_filter(wt, cout_p, cin_p)
    bias_p = torch.zeros(cout_p, device=DEV)
    bias_p[:cout] = bias
    y = torch.empty(batch, to, ho, wo, cout, device=DEV, dtype=torch.bfloat16)
    dyp = torch.empty(batch, t + kt - 1, h, w, cout_p, device=DEV, dtype=torch.bfloat16)
    db = torch.empty(cout, device=DEV)
    dxc = torch.empty(batch, t, h, w, cin, device=DEV, dtype=torch.bfloat16)
    dw = torch.empty(wt.shape, device=DEV)
    ours = {
        "pack_x": lambda: ops.conv3d_pack(xs, xp, t_offset=kt - 1),
        "pack_x_fp32": lambda: ops.conv3d_pack(xs32, xp, t_offset=kt - 1),     # GroupNorm's fp32 output under autocast
        "fwd": lambda: ops.causal_conv3d(xp, wf, bias_p, y, kernel=(k, k, k), stride=stride),
        "pack_dy_db": lambda: ops.conv3d_pack(dy, dyp, t_offset=0, dil=stride, bias_grad=db),
        "dgrad": lambda: ops.causal_conv3d(dyp, wb, None, dxc, kernel=(k, k, k)),
        "wgrad": lambda: ops.conv3d_wgrad(xp, dyp, dw, out_shape=(to, ho, wo), stride=stride),
        "filters": lambda: (VT.forward_filter(wt, cout_p, cin_p), VT.dgrad_filter(wt, cout_p, cin_p)),
    }
    # ---- torch: autocast conv3d on the padded input, cuDNN's data / weight gradients
    pad = (1, 1, 1, 1, 2, 0) if k == 3 else (0,) * 6
    xpad = F.pad(x, pad)
    wt16 = wt.bfloat16()
    conv_args = ([cout], list(stride), [0, 0, 0], [1, 1, 1], False, [0, 0, 0], 1)
    yt = F.conv3d(xpad, wt16, bias.bfloat16(), stride=stride)
    theirs = {
        "fwd": lambda: F.conv3d(xpad, wt16, bias.bfloat16(), stride=stride),
        "dgrad": lambda: torch.ops.aten.convolution_backward(dy, xpad, wt16, *conv_args, [True, False, False]),
        # the weight gradient alone: the library's bias gradient is part of its dy pack, timed on the pack_dy_db line
        "wgrad": lambda: torch.ops.aten.convolution_backward(dy, xpad, wt16, *conv_args, [False, True, False]),
    }
    times = {}
    for _ in range(2):          # alternate the two implementations
        for key, fn in ours.items():
            times.setdefault(("ours", key), []).append(timed(fn, iters, warmup))
        for key, fn in theirs.items():
            times.setdefault(("torch", key), []).append(timed(fn, iters, warmup))
    # outputs of both, compared
    for fn in ours.values():
        fn()
    dxt = torch.ops.aten.convolution_backward(dy, xpad, wt16, *conv_args, [True, False, False])[0]
    dwt = torch.ops.aten.convolution_backward(dy, xpad, wt16, *conv_args, [False, True, False])[1]
    if k == 3:
        dxt = dxt[:, :, 2:, 1:-1, 1:-1]
    diff = {"fwd": rel_rms(y.permute(0, 4, 1, 2, 3), yt), "dgrad": rel_rms(dxc.permute(0, 4, 1, 2, 3), dxt),
            "wgrad": rel_rms(dw, dwt)}
    rows = []
    for key in ("fwd", "dgrad", "wgrad"):
        mo, mt = statistics.median(times[("ours", key)]), statistics.median(times[("torch", key)])
        rows.append({"family": name, "pass": key, "cin": cin, "cout": cout, "k": k, "stride": list(stride),
                     "input_thw": list(thw), "batch": batch,
                     "ours_ms": round(mo, 4), "ours_tflops": round(flops / mo / 1e9, 1),
                     "cudnn_ms": round(mt, 4), "cudnn_tflops": round(flops / mt / 1e9, 1),
                     "speedup_vs_cudnn": round(mt / mo, 3), "rel_rms_vs_cudnn": float(f"{diff[key]:.3e}")})
    for key in ("pack_x", "pack_x_fp32", "pack_dy_db", "filters"):
        rows.append({"family": name, "pass": key, "ours_ms": round(statistics.median(times[("ours", key)]), 4)})
    # the kernels inside the wgrad and dy-pack calls on lines of their own (device time per call, torch.profiler, after the
    # timed runs): the weight-gradient GEMM and its split reduce; the pack and the two bias-gradient reduce passes
    for key, kernels in (("wgrad", ("conv3d_wgrad_kernel", "conv_wgrad_reduce_kernel")),
                         ("pack_dy_db", ("conv_pack_kernel", "conv_bias_grad_kernel"))):
        for kern, ms in kernel_ms(ours[key], kernels).items():
            rows.append({"family": name, "pass": f"{key}:{kern}", "ours_ms": round(ms, 4)})
    return rows


def kernel_ms(fn, names, reps: int = 5) -> dict:
    """Device time per call of each kernel whose name contains one of `names` (all launches of it in one call summed)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for evt in prof.key_averages():
        total_us = getattr(evt, "device_time_total", None)
        if total_us is None:
            total_us = evt.cuda_time_total
        for n in names:
            if n in evt.key:
                out[n] += total_us / 1e3 / reps
    return out


def _reference_vae():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        raise SystemExit("the reference's sources are not staged (oracle/_ref): run build() first")
    ref_shim.install()
    CausalVideoVAE = __import__("video_vae", fromlist=["CausalVideoVAE"]).CausalVideoVAE
    vae = CausalVideoVAE()          # full-size: (128, 256, 512, 512), latent 4, synthetic (trunc-normal) weights
    return vae.to(DEV).train()


def _step_fn(vae):
    params = [p for p in vae.parameters()]

    def step(x):
        for p in params:
            p.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            posterior, dec = vae(x, sample_posterior=True, generator=torch.Generator().manual_seed(0))
            loss = (dec.float() - x).abs().mean() + 1e-6 * posterior.kl().mean()
        loss.backward()
        return loss
    return step


STEP_INPUTS = {"video_b2_t17_256": (2, 3, 17, 256, 256), "images_b8_t1_256": (8, 3, 1, 256, 256)}
VARIANTS = {"torch": (), "library": (VT.install_training_convs,),
            "library_norms": (VT.install_training_convs, VT.install_training_norms)}


def _uninstall_all(vae):
    VT.uninstall_training_convs(vae)
    VT.uninstall_training_norms(vae)


def bench_step(vae, rounds: int, iters: int, warmup: int) -> list:
    step = _step_fn(vae)
    rows = []
    for name, shape in STEP_INPUTS.items():
        x = torch.randn(*shape, device=DEV)
        res = {v: [] for v in VARIANTS}
        peak, losses = {}, {}
        copies = 0
        for r in range(rounds):
            for variant, installs in VARIANTS.items():
                for inst in installs:
                    inst(vae)
                try:
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    n0 = VT.layout_copies
                    res[variant].append(timed(lambda: step(x), iters, warmup))
                    peak[variant] = max(peak.get(variant, 0), torch.cuda.max_memory_allocated())
                    losses[variant] = step(x).item()
                    if variant == "library_norms":
                        copies = (VT.layout_copies - n0) // (iters + warmup + 1)
                finally:
                    _uninstall_all(vae)
        med = {v: statistics.median(res[v]) for v in VARIANTS}
        rows.append({"step": name, "torch_ms": round(med["torch"], 2), "library_ms": round(med["library"], 2),
                     "library_norms_ms": round(med["library_norms"], 2), "speedup": round(med["torch"] / med["library"], 3),
                     "speedup_norms": round(med["torch"] / med["library_norms"], 3),
                     "norms_vs_convs_only": round(med["library"] / med["library_norms"], 3),
                     **{f"{v}_rounds_ms": [round(t, 2) for t in res[v]] for v in VARIANTS},
                     **{f"{v}_peak_gib": round(peak[v] / 2 ** 30, 2) for v in VARIANTS},
                     **{f"loss_{v}": losses[v] for v in VARIANTS},
                     "norm_layout_copies_per_step": copies,
                     "note": "L1 + KL only: LPIPS needs a checkpoint, the discriminator starts at step 250000"})
        del x
        torch.cuda.empty_cache()
    return rows


def _form_name(t) -> str:
    return ops.groupnorm_form(t) or "other"


def norm_sites(vae) -> dict:
    """(shape, input form, dtype, groups, gradient form) -> names of the CausalGroupNorm sites with such an input, over one
    video step with the convs and the norms installed; the gradient form is the layout the output's gradient arrives in
    (a site copies its input when the input form is "other", its gradient when the two forms differ)."""
    x_key, dy_form = {}, {}

    def pre_hook(name):
        def hook(mod, args):
            x = args[0]
            x_key[name] = (tuple(x.shape), _form_name(x), str(x.dtype).replace("torch.", ""), mod.num_groups)
        return hook

    def out_hook(name):
        def hook(mod, args, out):
            if out.requires_grad:
                out.register_hook(lambda g: dy_form.__setitem__(name, _form_name(g)))
        return hook

    norms = VT.causal_group_norms(vae)
    handles = [m.register_forward_pre_hook(pre_hook(n)) for n, m in norms]
    handles += [m.register_forward_hook(out_hook(n)) for n, m in norms]
    VT.install_training_convs(vae)
    VT.install_training_norms(vae)
    try:
        _step_fn(vae)(torch.randn(*STEP_INPUTS["video_b2_t17_256"], device=DEV))
    finally:
        _uninstall_all(vae)
        for h in handles:
            h.remove()
    torch.cuda.synchronize()
    sites = {}
    for name, key in x_key.items():
        sites.setdefault(key + (dy_form.get(name, "none"),), []).append(name)
    return sites


def _in_layout(t, form):
    return t.contiguous() if form == "plane" else t.contiguous(memory_format=torch.channels_last_3d)


def bench_norm_family(key, names, iters, warmup) -> dict:
    """One norm family, x and dy in the layouts the step delivers (a gradient in the other form than x is copied inside
    causal_group_norm's backward, and the copy is part of the timing)."""
    shape, form, dtype, groups, dy_form = key
    g = torch.Generator(device=DEV).manual_seed(0)
    x = _in_layout(torch.randn(*shape, device=DEV, generator=g).to(getattr(torch, dtype)), form)
    c = shape[1]
    gamma = (1 + 0.2 * torch.randn(c, device=DEV, generator=g)).requires_grad_(True)
    beta = (0.1 * torch.randn(c, device=DEV, generator=g)).requires_grad_(True)
    dy = _in_layout(torch.randn(*shape, device=DEV, generator=g, dtype=torch.bfloat16), dy_form)
    xr = x.detach().requires_grad_(True)
    silu = torch.nn.SiLU()

    def ours_fwd():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return VT.causal_group_norm(xr, gamma, beta, groups, 1e-6, silu=True, out_dtype=torch.bfloat16)

    def ref_fwd():
        b, _, t, h, w = shape
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = torch.nn.functional.group_norm(xr.transpose(1, 2).reshape(b * t, c, h, w), groups, gamma, beta, 1e-6)
            return silu(y.reshape(b, t, c, h, w).transpose(1, 2))

    def fwd_bwd(fn):
        # the gradients are returned, not accumulated into xr.grad: accumulating a channels-last dx into an NCDHW leaf
        # makes torch copy it into the leaf's layout, which is not part of the op (in the step, dx flows on upstream)
        return lambda: torch.autograd.grad(fn(), (xr, gamma, beta), dy)

    times = {}
    for _ in range(2):
        for name, fn in (("ours_fwd", ours_fwd), ("ref_fwd", ref_fwd), ("ours_fwd_bwd", fwd_bwd(ours_fwd)),
                         ("ref_fwd_bwd", fwd_bwd(ref_fwd))):
            times.setdefault(name, []).append(timed(fn, iters, warmup))
    xr.grad = None
    yo = ours_fwd()
    yo.backward(dy)
    dxo = xr.grad.clone()
    xr.grad = None
    yr = ref_fwd()
    yr.backward(dy.float())
    dxr = xr.grad.clone()
    med = {k: statistics.median(v) for k, v in times.items()}
    numel = x.numel()
    return {"norm_family": list(shape), "form": form, "dtype": dtype, "groups": groups, "dy_form": dy_form,
            "sites_per_step": len(names), "sites": names,
            "ours_fwd_ms": round(med["ours_fwd"], 4), "torch_fwd_ms": round(med["ref_fwd"], 4),
            "ours_fwd_bwd_ms": round(med["ours_fwd_bwd"], 4), "torch_fwd_bwd_ms": round(med["ref_fwd_bwd"], 4),
            "speedup_fwd": round(med["ref_fwd"] / med["ours_fwd"], 3),
            "speedup_fwd_bwd": round(med["ref_fwd_bwd"] / med["ours_fwd_bwd"], 3),
            "ours_fwd_GBps": round(numel * (2 * x.element_size() + 2) / med["ours_fwd"] / 1e6, 1),
            "rel_rms_y_vs_torch": float(f"{rel_rms(yo, yr.bfloat16()):.3e}"),
            "rel_rms_dx_vs_torch": float(f"{rel_rms(dxo, dxr):.3e}"),
            "note": "torch: reference CausalGroupNorm math + nn.SiLU under bf16 autocast (fp32 output); ours: bf16 output"}


PROFILED_OPS = ("aten::native_group_norm", "aten::native_group_norm_backward", "aten::silu", "aten::silu_backward",
                "aten::silu_")


def profile_steps(vae) -> list:
    """Device time per step of torch's GroupNorm / SiLU ops and of the conv pack kernel, convs-only vs convs + norms."""
    from torch.profiler import ProfilerActivity, profile
    step = _step_fn(vae)
    x = torch.randn(*STEP_INPUTS["video_b2_t17_256"], device=DEV)
    rows = []
    for variant in ("library", "library_norms"):
        for inst in VARIANTS[variant]:
            inst(vae)
        try:
            step(x)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                step(x)
                torch.cuda.synchronize()
        finally:
            _uninstall_all(vae)
        row = {"profile_step": "video_b2_t17_256", "variant": variant}
        kernels = {"conv_pack_kernel": 0.0, "gt_": 0.0}
        for evt in prof.key_averages():
            dev_us = getattr(evt, "device_time_total", None)
            if dev_us is None:
                dev_us = evt.cuda_time_total
            if evt.key in PROFILED_OPS:
                row[f"{evt.key}_ms"] = round(dev_us / 1e3, 3)
                row[f"{evt.key}_calls"] = evt.count
            for k in kernels:
                if k in evt.key and "aten::" not in evt.key:
                    kernels[k] += getattr(evt, "self_device_time_total", dev_us) / 1e3
        row["conv_pack_kernel_ms"] = round(kernels["conv_pack_kernel"], 3)
        row["library_norm_kernels_ms"] = round(kernels["gt_"], 3)
        rows.append(row)
    return rows


# ---- LPIPS -----------------------------------------------------------------------------------------------------------
LPIPS_SHAPES = {"clip_34+34_256": (34, 256), "images_8+8_256": (8, 256)}


def vgg_flop(n: int, hw: int, first_cin: int = 3) -> float:
    """Algorithmic FLOP of VGG16 features[:30] (up to relu5_3) on n images of hw x hw."""
    total, size = 0.0, hw
    for s, idx in enumerate(((0, 1), (2, 3), (4, 5, 6), (7, 8, 9), (10, 11, 12))):
        if s:
            size //= 2
        for i in idx:
            cin, cout = VT.VGG16_CONVS[i]
            total += 2.0 * size * size * (first_cin if i == 0 else cin) * cout * 9
    return n * total


def _lpips_module(seed: int = 0):
    from oracle.pin import ref_shim
    ref_shim.install()
    import io
    import warnings
    from tests.test_train_lpips_cpu import synthetic_lpips_state
    buf = io.BytesIO()
    torch.save(synthetic_lpips_state(seed), buf)
    path = Path(__import__("tempfile").mkdtemp()) / "lpips.pth"
    path.write_bytes(buf.getvalue())
    loss_cls = __import__("video_vae.modeling_loss", fromlist=["LPIPSWithDiscriminator"]).LPIPSWithDiscriminator
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        loss = loss_cls(disc_start=250000, kl_weight=1e-12, pixelloss_weight=10.0, perceptual_weight=1.0,
                        lpips_ckpt=str(path))
    path.unlink()
    return loss.to(DEV).train()


def bench_lpips(iters: int, warmup: int) -> list:
    lp = _lpips_module().perceptual_loss.train()
    rows = []
    for name, (n, hw) in LPIPS_SHAPES.items():
        g = torch.Generator(device=DEV).manual_seed(n)
        x0 = torch.rand(n, 3, hw, hw, device=DEV, generator=g) * 2 - 1
        x1 = (x0 + 0.2 * torch.randn(n, 3, hw, hw, device=DEV, generator=g)).clamp(-1, 1)

        def ours_fwd():
            with torch.no_grad():
                return VT.lpips(x0, x1, lp)

        def ref_fwd():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                return lp(x0, x1)

        def fwd_bwd(fn_lib):
            def run():
                xr = x1.clone().requires_grad_(True)
                if fn_lib:
                    v = VT.lpips(x0, xr, lp)
                else:
                    with torch.autocast("cuda", dtype=torch.bfloat16):
                        v = lp(x0, xr)
                v.float().sum().backward()
                return xr.grad
            return run

        f_flop, b_flop = vgg_flop(2 * n, hw), vgg_flop(n, hw)
        row = {"lpips": name, "images_per_branch": n}
        for key, fn, flop in (("fwd", (ours_fwd, ref_fwd), f_flop),
                              ("fwd_bwd", (fwd_bwd(True), fwd_bwd(False)), f_flop + b_flop)):
            for who, f in zip(("library", "torch"), fn):
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                ms = timed(f, iters, warmup)
                row[f"{key}_{who}_ms"] = round(ms, 3)
                row[f"{key}_{who}_peak_gib"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)
                row[f"{key}_{who}_tflops"] = round(flop / ms / 1e9, 1)
            row[f"{key}_speedup"] = round(row[f"{key}_torch_ms"] / row[f"{key}_library_ms"], 3)
        row["algorithmic_tflop_fwd"] = round(f_flop / 1e12, 3)
        row["algorithmic_tflop_dgrad"] = round(b_flop / 1e12, 3)
        lp.eval()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            row["rel_rms_eval_value_vs_torch"] = rel_rms(VT.lpips(x0, x1, lp), lp(x0, x1))
        lp.train()
        rows.append(row)

        # the first conv alone: 3 channels padded to 64 in the packed input
        conv = lp.net.slice1[0]
        xp = torch.zeros(2 * n, 1, hw, hw, 64, device=DEV, dtype=torch.bfloat16)
        y = torch.empty(2 * n, 1, hw, hw, 64, device=DEV, dtype=torch.bfloat16)
        wf, bias = VT._vgg_filter(conv.weight), VT._vgg_bias(conv.bias)
        ms = timed(lambda: ops.causal_conv3d(xp, wf, bias, y, kernel=(1, 3, 3), relu=True), iters, warmup)
        real = 2.0 * 2 * n * hw * hw * 3 * 64 * 9
        rows.append({"lpips_first_conv": name, "images": 2 * n, "ms": round(ms, 3),
                     "padded_tflop": round(real * 64 / 3 / 1e12, 3), "real_tflop": round(real / 1e12, 4),
                     "padded_work_over_real": round(64 / 3, 1), "padded_tflops": round(real * 64 / 3 / ms / 1e9, 1)})

        fams = {"conv3d_wgmma_kernel": 0.0, "maxpool2x2_kernel": 0.0, "lpips_head": 0.0, "lpips_tap_bwd_kernel": 0.0,
                "conv_pack_kernel": 0.0}
        f_only = kernel_ms(ours_fwd, list(fams))
        both = kernel_ms(fwd_bwd(True), list(fams))
        rows.append({"lpips_profile": name, "vgg_convs_fwd_ms": round(f_only["conv3d_wgmma_kernel"], 3),
                     "dgrad_convs_ms": round(both["conv3d_wgmma_kernel"] - f_only["conv3d_wgmma_kernel"], 3),
                     "pool_ms": round(both["maxpool2x2_kernel"], 3), "head_fwd_ms": round(both["lpips_head"], 3),
                     "tap_bwd_ms": round(both["lpips_tap_bwd_kernel"], 3), "input_pack_ms": round(both["conv_pack_kernel"], 3)})
        del x0, x1, xp, y
        torch.cuda.empty_cache()
    return rows


LOSS_VARIANTS = {"torch": (), "library_norms": (VT.install_training_convs, VT.install_training_norms),
                 "library_norms_lpips": (VT.install_training_convs, VT.install_training_norms, VT.install_training_lpips)}


def bench_step_lpips(vae, rounds: int, iters: int, warmup: int) -> list:
    """The generator step with LPIPSWithDiscriminator (optimizer_idx 0, before disc_start)."""
    class Step(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.vae, self.loss = vae, _lpips_module()

    model = Step().train()
    params = list(model.parameters())

    def step(x):
        for p in params:
            p.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            posterior, dec = vae(x, sample_posterior=True, generator=torch.Generator().manual_seed(0))
            loss, _ = model.loss(x, dec, posterior, optimizer_idx=0, global_step=0, last_layer=vae.get_last_layer())
        loss.backward()
        return loss

    rows = []
    for name, shape in STEP_INPUTS.items():
        x = torch.rand(*shape, device=DEV) * 2 - 1
        res = {v: [] for v in LOSS_VARIANTS}
        peak, losses = {}, {}
        for _ in range(rounds):
            for variant, installs in LOSS_VARIANTS.items():
                for inst in installs:
                    inst(model)
                try:
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    res[variant].append(timed(lambda: step(x), iters, warmup))
                    peak[variant] = max(peak.get(variant, 0), torch.cuda.max_memory_allocated())
                    losses[variant] = step(x).item()
                finally:
                    VT.uninstall_training_lpips(model)
                    _uninstall_all(vae)
        med = {v: statistics.median(res[v]) for v in LOSS_VARIANTS}
        rows.append({"step_with_lpips_loss": name, **{f"{v}_ms": round(med[v], 2) for v in LOSS_VARIANTS},
                     "speedup_norms": round(med["torch"] / med["library_norms"], 3),
                     "speedup_norms_lpips": round(med["torch"] / med["library_norms_lpips"], 3),
                     **{f"{v}_rounds_ms": [round(t, 2) for t in res[v]] for v in LOSS_VARIANTS},
                     **{f"{v}_peak_gib": round(peak[v] / 2 ** 30, 2) for v in LOSS_VARIANTS},
                     **{f"loss_{v}": losses[v] for v in LOSS_VARIANTS},
                     "note": "pixel 10 + LPIPS 1 (dropout live) + KL 1e-12; the discriminator starts at step 250000"})
        del x
        torch.cuda.empty_cache()
    return rows


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--step-iters", type=int, default=3)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--skip-families", action="store_true")
    ap.add_argument("--skip-norms", action="store_true")
    ap.add_argument("--skip-profile", action="store_true")
    ap.add_argument("--skip-lpips", action="store_true")
    args = ap.parse_args()
    _lib.require_device()
    print(json.dumps(device_info()), flush=True)
    if not args.skip_families:
        for fam in FAMILIES:
            for row in bench_family(*fam, iters=args.iters, warmup=args.warmup):
                print(json.dumps(row), flush=True)
            torch.cuda.empty_cache()
    if not args.skip_lpips:
        for row in bench_lpips(args.iters, args.warmup):
            print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()
    vae = None if (args.skip_step and args.skip_norms and args.skip_profile and args.skip_lpips) else _reference_vae()
    if not args.skip_norms:
        for key, names in sorted(norm_sites(vae).items(), key=lambda kv: -kv[0][0][1]):
            print(json.dumps(bench_norm_family(key, names, args.iters, args.warmup)), flush=True)
            torch.cuda.empty_cache()
    if not args.skip_step:
        for row in bench_step(vae, args.rounds, args.step_iters, 1):
            print(json.dumps(row), flush=True)
    if not args.skip_lpips:
        for row in bench_step_lpips(vae, args.rounds, args.step_iters, 1):
            print(json.dumps(row), flush=True)
    if not args.skip_profile:
        for row in profile_steps(vae):
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
