"""Training GroupNorm (+ SiLU) of the causal video VAE on the GPU: causal_group_norm's output and its x / weight / bias
gradients against fp64 autograd of the reference's CausalGroupNorm (+ SiLU) on the same rounded inputs (relative RMS error
within 1.5x of torch's group_norm under bf16 autocast against the same fp64 result), bit equality with the inference
kernels, bitwise repeatability (also under checkpoint recompute), what the autograd function saves, and a tiny unmodified
reference CausalVideoVAE trained one step with install_training_norms, alone and with install_training_convs."""
import contextlib
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from pyramid_flow_b200 import _lib, ops
from pyramid_flow_b200 import vae_training as VT
from tests.test_train_vae_conv_cpu import TINY_VAE, _reference_vae_cls
from tests.test_train_vae_norm_cpu import _reference_norm

pytestmark = pytest.mark.gpu

RATIO = 1.5
FLOOR = 1e-7          # fp32 rounding noise: a case whose torch error is ~0 (the constant input) may not be held to 0
EPS = 1e-6


def _rel_rms(a, ref):
    a, ref = a.double(), ref.double()
    return ((a - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt().clamp_min(1e-30)).item()


def _layout(x, form):
    if form == "channel":
        return x.contiguous(memory_format=torch.channels_last_3d)
    if form == "plane":
        return x.contiguous()
    if form == "plane_bt":        # the mid-block attention's (b t) c h w -> b c t h w view: planes with permuted strides
        return x.permute(0, 2, 1, 3, 4).contiguous().permute(0, 2, 1, 3, 4)
    if form == "fallback":        # a W-sliced view: neither form, copied to channels_last_3d
        b, c, t, h, w = x.shape
        big = torch.empty(b, c, t, h, w + 8, device=x.device, dtype=x.dtype)
        big[..., :w] = x
        return big[..., :w]
    raise ValueError(form)


CASES = [
    # c, b, t, h, w, form, dtype, silu, out_bf16
    (64, 2, 5, 24, 40, "channel", torch.bfloat16, True, True),
    (128, 1, 1, 24, 40, "channel", torch.bfloat16, False, False),
    (256, 2, 9, 72, 100, "channel", torch.float32, True, False),      # 7200 voxels: 2 splits
    (512, 1, 17, 16, 24, "channel", torch.bfloat16, True, False),
    (64, 2, 5, 24, 40, "channel", torch.float32, False, True),
    (64, 2, 17, 24, 40, "plane", torch.bfloat16, True, True),
    (128, 1, 5, 72, 100, "plane", torch.float32, False, False),
    (256, 2, 1, 130, 90, "plane", torch.bfloat16, True, False),        # 11700 voxels: 3 splits
    (512, 2, 9, 12, 20, "plane", torch.float32, True, True),
    (64, 1, 5, 15, 13, "plane", torch.bfloat16, True, False),          # 195 voxels: element loads
    (128, 2, 9, 70, 64, "plane_bt", torch.bfloat16, True, True),
    (128, 2, 5, 24, 40, "fallback", torch.bfloat16, True, False),
    (64, 2, 5, 24, 40, "fallback", torch.float32, False, True),
]


def _case_id(c):
    return f"c{c[0]}_b{c[1]}_t{c[2]}_{c[3]}x{c[4]}_{c[5]}_{str(c[6])[6:]}_{'silu' if c[7] else 'nosilu'}_{'obf16' if c[8] else 'of32'}"


def _inputs(c, b, t, h, w, dtype, seed, shift=0.0, constant=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(b, c, t, h, w, device="cuda", generator=g) * 1.5 + 0.3
    if shift:
        x = x + shift * 1.5
    if constant:
        x = torch.full_like(x, 0.75)
    gamma = 1 + 0.3 * torch.randn(c, device="cuda", generator=g)
    beta = 0.2 * torch.randn(c, device="cuda", generator=g)
    dy = torch.randn(b, c, t, h, w, device="cuda", generator=g)
    return x.to(dtype), gamma, beta, dy


def _check(c, b, t, h, w, form, dtype, silu, out_bf16, *, seed=0, shift=0.0, constant=False, dy_form=None, copies=None):
    groups = 32
    x, gamma, beta, dy = _inputs(c, b, t, h, w, dtype, seed, shift, constant)
    xl = _layout(x, form)
    # dy in the layout of the output (or dy_form), as the next conv's backward hands it over
    dy = _layout(dy.bfloat16() if out_bf16 else dy, dy_form or ("plane" if form.startswith("plane") else "channel"))

    # fp64 autograd of the reference on the same rounded inputs
    x64 = x.double().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    y64 = _reference_norm(x64, g64, b64, groups, EPS, silu)
    y64.backward(dy.double())

    # torch: group_norm (+ SiLU) under bf16 autocast, its autograd
    xt = xl.detach().clone().requires_grad_(True)
    gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        yt = _reference_norm(xt, gt, bt, groups, EPS, silu)
    assert yt.dtype == torch.float32
    yt.backward(dy.to(yt.dtype))

    n0 = VT.layout_copies
    xo = xl.detach().requires_grad_(True)
    go, bo = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        yo = VT.causal_group_norm(xo, go, bo, groups, EPS, silu=silu, out_dtype=torch.bfloat16 if out_bf16 else None)
    assert yo.dtype == (torch.bfloat16 if out_bf16 else torch.float32) and yo.shape == x.shape
    if form == "channel" or form == "fallback":
        assert yo.is_contiguous(memory_format=torch.channels_last_3d)
    else:
        assert yo.is_contiguous()
    yo.backward(dy)
    assert VT.layout_copies - n0 == (copies if copies is not None else (1 if form == "fallback" else 0))
    assert xo.grad.dtype == x.dtype and go.grad.dtype == torch.float32

    ref_t = yt.detach().bfloat16() if out_bf16 else yt.detach()
    pairs = [("y", yo.detach(), ref_t, y64.detach()), ("dx", xo.grad, xt.grad, x64.grad),
             ("dgamma", go.grad, gt.grad, g64.grad), ("dbeta", bo.grad, bt.grad, b64.grad)]
    for name, ours, theirs, ref in pairs:
        e_o, e_t = _rel_rms(ours, ref), _rel_rms(theirs, ref)
        assert e_o <= RATIO * e_t + FLOOR, (name, e_o, e_t)
    return yo.detach(), xo.grad, go.grad, bo.grad


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_causal_group_norm_vs_fp64(case):
    _check(*case)


@pytest.mark.parametrize("c, dtype", [(128, torch.bfloat16), (512, torch.bfloat16), (96, torch.bfloat16),
                                      (128, torch.float32)])
@pytest.mark.parametrize("form", ["plane", "plane_bt"])
def test_plane_input_with_a_channels_last_gradient(c, dtype, form):
    """The sites after the up-samplers: x has planes, the next conv's data gradient arrives channels_last_3d.  A bf16 x
    with channels a multiple of 64 is repacked channels-last (pf_conv3d_pack), otherwise dy is copied into planes: one
    copy either way, and the same accuracy."""
    _check(c, 2, 5, 40, 48, form, dtype, True, True, seed=9, dy_form="channel", copies=1)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("form", ["channel", "plane"])
def test_large_mean_against_std(dtype, form):
    """|mean| / std = 100: the pivot-shifted sums keep the variance."""
    _check(128, 2, 5, 40, 48, form, dtype, True, False, seed=3, shift=100.0)


@pytest.mark.parametrize("form", ["channel", "plane"])
def test_constant_input(form):
    """var = 0: rstd = 1/sqrt(eps), the output is act(beta), finite gradients."""
    y, dx, dg, db = _check(64, 1, 3, 16, 16, form, torch.bfloat16, True, False, seed=4, constant=True)
    assert torch.isfinite(dx.float()).all() and torch.isfinite(dg).all() and torch.isfinite(db).all()


def test_bit_equality_with_the_inference_kernels():
    """A bf16 channels-last input: the same (mean, rstd) and the same bf16 SiLU output as pf_groupnorm_stats + apply."""
    b, c, t, h, w, groups = 2, 128, 5, 72, 100, 32
    x, gamma, beta, _ = _inputs(c, b, t, h, w, torch.bfloat16, 8)
    x = x.contiguous(memory_format=torch.channels_last_3d)
    frames, voxels = b * t, h * w
    stats = torch.empty(frames, groups, 2, device="cuda")
    y = torch.empty(b, t, h, w, c, device="cuda", dtype=torch.bfloat16).permute(0, 4, 1, 2, 3)
    ops.groupnorm_train_fwd(x, gamma, beta, stats, y, groups=groups, eps=EPS, silu=True)

    lib = _lib.load()
    ws = torch.empty(frames * 64 * c * 2, device="cuda")
    stats_i = torch.empty(frames, groups, 2, device="cuda")
    y_i = torch.empty(frames, voxels, c, device="cuda", dtype=torch.bfloat16)
    _lib.check(lib.pf_groupnorm_stats(x.data_ptr(), frames, voxels, c, groups, EPS, stats_i.data_ptr(), ws.data_ptr(),
                                      ws.numel(), _lib.stream_ptr()), "pf_groupnorm_stats")
    _lib.check(lib.pf_groupnorm_apply(x.data_ptr(), y_i.data_ptr(), 1, frames, voxels, c, groups, stats_i.data_ptr(),
                                      gamma.data_ptr(), beta.data_ptr(), 1, frames, 0, _lib.stream_ptr()), "pf_groupnorm_apply")
    assert torch.equal(stats, stats_i)
    assert torch.equal(y.permute(0, 2, 3, 4, 1).reshape(frames, voxels, c), y_i)


@pytest.mark.parametrize("form", ["channel", "plane"])
def test_determinism_and_checkpoint_recompute(form):
    x, gamma, beta, dy = _inputs(256, 2, 9, 72, 100, torch.bfloat16, 5)
    x = _layout(x, form)
    dy = dy.bfloat16()

    def run(checkpointed):
        xo = x.detach().requires_grad_(True)
        go, bo = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        fn = lambda a, g_, b_: VT.causal_group_norm(a, g_, b_, 32, EPS, silu=True, out_dtype=torch.bfloat16)  # noqa: E731
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = torch.utils.checkpoint.checkpoint(fn, xo, go, bo, use_reentrant=False) if checkpointed else fn(xo, go, bo)
        y.backward(dy)
        return y.detach(), xo.grad, go.grad, bo.grad

    a, b_, c = run(False), run(False), run(True)
    for u, v, w in zip(a, b_, c):
        assert torch.equal(u, v) and torch.equal(u, w)


@pytest.mark.parametrize("form", ["channel", "plane"])
def test_saved_tensors_are_x_and_the_statistics(form):
    x, gamma, beta, _ = _inputs(128, 2, 5, 32, 32, torch.bfloat16, 6)
    x = _layout(x, form).requires_grad_(True)
    w, b = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    saved = []

    def pack(t):
        saved.append(t)
        return t

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = VT.causal_group_norm(x, w, b, 32, EPS, silu=True, out_dtype=torch.bfloat16)
    big = [t for t in saved if t.numel() >= x.numel() // 4]
    assert len(big) == 1 and big[0].data_ptr() == x.data_ptr() and big[0].dtype == torch.bfloat16   # x itself, no copy
    small = [t for t in saved if t.numel() < x.numel() // 4]
    assert any(t.shape == (2 * 5, 32, 2) and t.dtype == torch.float32 for t in small)
    assert len(saved) == 4                  # x, weight, bias, stats
    y.float().sum().backward()


def _to_channels_last_on_unpack():
    """A saved-tensor hook that hands 5-D tensors back channels_last_3d (the other direction from save_on_cpu's)."""
    def unpack(t):
        return t.contiguous(memory_format=torch.channels_last_3d) if t.dim() == 5 else t
    return torch.autograd.graph.saved_tensors_hooks(lambda t: t, unpack)


@pytest.mark.parametrize("hook", ["save_on_cpu_pinned", "save_on_cpu", "channels_last_on_unpack"])
@pytest.mark.parametrize("form", ["channel", "plane", "plane_bt"])
def test_saved_tensor_hooks_that_change_strides(form, hook):
    """save_on_cpu unpacks x as a contiguous NCDHW tensor: the backward must still run, with the gradients of a plain run
    bit for bit."""
    x, gamma, beta, dy = _inputs(128, 2, 5, 32, 40, torch.bfloat16, 7)
    x = _layout(x, form)
    dy = _layout(dy.bfloat16(), "plane" if form.startswith("plane") else "channel")

    def run(ctx):
        xo = x.detach().requires_grad_(True)
        go, bo = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        with ctx:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = VT.causal_group_norm(xo, go, bo, 32, EPS, silu=True, out_dtype=torch.bfloat16)
        y.backward(dy)
        return y.detach(), xo.grad, go.grad, bo.grad

    plain = run(contextlib.nullcontext())
    ctx = {"save_on_cpu_pinned": lambda: torch.autograd.graph.save_on_cpu(pin_memory=True),
           "save_on_cpu": lambda: torch.autograd.graph.save_on_cpu(pin_memory=False),
           "channels_last_on_unpack": _to_channels_last_on_unpack}[hook]()
    hooked = run(ctx)
    for name, a, b in zip(("y", "dx", "dgamma", "dbeta"), plain, hooked):
        assert torch.equal(a, b), name


# ---- the drop-in on a tiny unmodified reference CausalVideoVAE ------------------------------------------------------------
@pytest.fixture(autouse=True)
def _deterministic_torch(monkeypatch):
    from torch.nn.attention import SDPBackend, sdpa_kernel
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    with sdpa_kernel(SDPBackend.MATH):
        yield


def _vae(seed=11):
    vae = _reference_vae_cls()(**TINY_VAE)
    from oracle.pin import ref_shim
    ref_shim.reinit_all_parameters(vae, seed=seed, std=0.05)
    # the reinit draws the norms' affine parameters around 0 as well: give them the scale of trained ones
    g = torch.Generator().manual_seed(seed)
    for _, m in VT.causal_group_norms(vae):
        with torch.no_grad():
            m.weight.copy_(1 + 0.2 * torch.randn(m.weight.shape, generator=g))
    return vae.cuda().train()


def _step(vae, x, *, autocast: bool, freeze_encoder=False):
    vae.zero_grad(set_to_none=True)
    gen = torch.Generator().manual_seed(5)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        posterior, dec = vae(x, sample_posterior=True, generator=gen, freeze_encoder=freeze_encoder)
        loss = (dec.float() - x).abs().mean() + 1e-3 * posterior.kl().mean()
    loss.backward()
    return loss.detach(), {n: p.grad.detach().clone() for n, p in vae.named_parameters() if p.grad is not None}


def _install(vae, which):
    VT.install_training_norms(vae)
    if which == "convs+norms":
        VT.install_training_convs(vae)


def _uninstall(vae):
    VT.uninstall_training_convs(vae)
    VT.uninstall_training_norms(vae)


@pytest.mark.parametrize("which", ["norms", "convs+norms"])
@pytest.mark.parametrize("frames", [9, 1])
@pytest.mark.parametrize("checkpointing", [False, True])
@pytest.mark.parametrize("freeze_encoder", [False, True])
def test_tiny_vae_training_step(which, frames, checkpointing, freeze_encoder):
    if freeze_encoder and checkpointing:
        pytest.skip("freeze_encoder runs the encoder under no_grad: checkpointing changes nothing there")
    vae = _vae()
    for p in list(vae.encoder.parameters()) + list(vae.quant_conv.parameters()):
        p.requires_grad_(not freeze_encoder)
    vae.encoder.gradient_checkpointing = checkpointing
    x = torch.randn(2, 3, frames, 32, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(frames))
    fe = dict(freeze_encoder=freeze_encoder)
    loss32, g32 = _step(vae, x, autocast=False, **fe)
    loss_t, g_t = _step(vae, x, autocast=True, **fe)
    _install(vae, which)
    try:
        loss_o, g_o = _step(vae, x, autocast=True, **fe)
        loss_o2, g_o2 = _step(vae, x, autocast=True, **fe)
    finally:
        _uninstall(vae)
    assert set(g_o) == set(g_t) == set(g32)
    e_loss_o, e_loss_t = abs(loss_o.item() - loss32.item()), abs(loss_t.item() - loss32.item())
    assert e_loss_o <= RATIO * e_loss_t + 1e-4 * abs(loss32.item()), (e_loss_o, e_loss_t)
    worse = []
    for n in g32:
        e_o, e_t = _rel_rms(g_o[n], g32[n]), _rel_rms(g_t[n], g32[n])
        if e_o > RATIO * e_t + 1e-4:
            worse.append((n, e_o, e_t))
    assert not worse, worse
    assert torch.equal(loss_o, loss_o2) and all(torch.equal(g_o[n], g_o2[n]) for n in g_o)


@pytest.mark.parametrize("which", ["norms", "convs+norms"])
def test_last_layer_grad_then_backward_matches_one_backward(which):
    """LPIPSWithDiscriminator.calculate_adaptive_weight (video_vae/modeling_loss.py:89-96): autograd.grad with
    retain_graph=True, twice, before the step's backward."""
    vae = _vae(seed=13)
    _install(vae, which)
    x = torch.randn(1, 3, 5, 32, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    try:
        _, plain = _step(vae, x, autocast=True)
        vae.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            posterior, dec = vae(x, sample_posterior=True, generator=torch.Generator().manual_seed(5))
            rec = (dec.float() - x).abs().mean()
            loss = rec + 1e-3 * posterior.kl().mean()
        last = vae.get_last_layer()
        g1 = torch.autograd.grad(rec, last, retain_graph=True)[0]
        g2 = torch.autograd.grad(loss, last, retain_graph=True)[0]
        assert torch.isfinite(g1).all() and torch.isfinite(g2).all()
        loss.backward()
        again = {n: p.grad for n, p in vae.named_parameters() if p.grad is not None}
    finally:
        _uninstall(vae)
    assert set(again) == set(plain)
    for n in plain:
        assert torch.equal(again[n], plain[n]), n


def test_uninstall_gives_the_reference_bits_again():
    vae = _vae(seed=17)
    x = torch.randn(1, 3, 5, 32, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    loss_a, g_a = _step(vae, x, autocast=True)
    VT.install_training_norms(vae)
    loss_i, _ = _step(vae, x, autocast=True)
    VT.uninstall_training_norms(vae)
    loss_b, g_b = _step(vae, x, autocast=True)
    assert not torch.equal(loss_i, loss_a)
    assert torch.equal(loss_a, loss_b) and all(torch.equal(g_a[n], g_b[n]) for n in g_a)
