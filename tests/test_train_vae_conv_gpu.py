"""Training convolutions of the causal video VAE on the GPU: causal_conv3d's output and its x / weight / bias gradients
against fp64 autograd of the reference's F.pad + conv3d on the same bf16-rounded operands (relative RMS error within 1.5x
of torch's bf16 autocast conv against the same fp64 result, and bitwise repeatable), and a tiny unmodified reference
CausalVideoVAE trained one step with and without install_training_convs."""
import pytest
import torch
import torch.nn.functional as F

from pyramid_flow_b200 import vae_training as VT
from tests.test_train_vae_conv_cpu import TINY_VAE, _reference_conv, _reference_vae_cls

pytestmark = pytest.mark.gpu

RATIO = 1.5


def _rel_rms(a, ref):
    a, ref = a.double(), ref.double()
    return ((a - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt().clamp_min(1e-30)).item()


CASES = [
    # cin, cout, k, stride, t, h, w, need_dx
    (3, 64, 3, (1, 1, 1), 5, 24, 40, False),      # conv_in on pixels: no dx
    (64, 64, 3, (1, 1, 1), 5, 24, 40, True),
    (64, 64, 3, (1, 1, 1), 1, 24, 40, True),
    (64, 128, 3, (1, 1, 1), 5, 24, 40, True),
    (64, 128, 1, (1, 1, 1), 5, 24, 40, True),      # resnet shortcut
    (128, 128, 3, (1, 2, 2), 5, 24, 40, True),
    (128, 128, 3, (1, 2, 2), 4, 20, 36, True),
    (128, 128, 3, (2, 1, 1), 1, 24, 40, True),
    (128, 128, 3, (2, 1, 1), 5, 24, 40, True),
    (128, 128, 3, (2, 1, 1), 4, 20, 36, True),
    (128, 32, 3, (1, 1, 1), 5, 24, 40, True),      # encoder conv_out (double_z, latent 16)
    (32, 32, 1, (1, 1, 1), 5, 24, 40, True),       # quant_conv
    (16, 128, 3, (1, 1, 1), 5, 24, 40, True),      # decoder conv_in
    (128, 512, 3, (1, 1, 1), 3, 24, 40, True),     # spatial up-sampler conv (x4 channels)
    (64, 3, 3, (1, 1, 1), 5, 24, 40, True),        # decoder conv_out
    (256, 256, 3, (1, 1, 1), 3, 24, 40, True),     # two 128-channel tiles of M and N in the weight gradient
    (512, 512, 3, (1, 1, 1), 2, 16, 24, True),
    (192, 192, 3, (1, 1, 1), 3, 20, 36, True),     # odd number of 64-channel boxes: the last tile has one dy / one x box
]


def _run_ours(x, w, b, stride, dy):
    x = x.detach().requires_grad_(x.requires_grad)
    w = w.detach().requires_grad_(True)
    b = b.detach().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = VT.causal_conv3d(x, w, b, stride)
    assert y.dtype == torch.bfloat16 and y.is_contiguous(memory_format=torch.channels_last_3d)
    y.backward(dy)
    return y.detach(), (x.grad if x.requires_grad else None), w.grad, b.grad


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}to{c[1]}_k{c[2]}_s{''.join(map(str, c[3]))}_t{c[4]}_{c[5]}x{c[6]}")
def test_causal_conv3d_parity_and_determinism(case):
    cin, cout, k, stride, t, h, w, need_dx = case
    g = torch.Generator(device="cuda").manual_seed(cin * 7 + cout + t)
    dev = torch.device("cuda")
    x = torch.randn(2, cin, t, h, w, device=dev, generator=g)
    wt = torch.randn(cout, cin, k, k, k, device=dev, generator=g) * (1.0 / (cin * k ** 3) ** 0.5)
    b = torch.randn(cout, device=dev, generator=g) * 0.1
    x.requires_grad_(need_dx)
    to, ho, wo = VT._out_dims(x.shape, stride)
    dy = torch.randn(2, cout, to, ho, wo, device=dev, generator=g).bfloat16()

    # fp64 autograd of the reference on the same bf16-rounded operands
    x64 = x.detach().bfloat16().double().requires_grad_(need_dx)
    w64 = wt.detach().bfloat16().double().requires_grad_(True)
    b64 = b.detach().double().requires_grad_(True)
    y64 = _reference_conv(x64, w64, b64, stride)
    y64.backward(dy.double())

    # torch's bf16 autocast conv (cuDNN) + autograd
    xt = x.detach().requires_grad_(need_dx)
    wtt = wt.detach().requires_grad_(True)
    bt = b.detach().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        yt = _reference_conv(xt, wtt, bt, stride)
    yt.backward(dy)

    y1, dx1, dw1, db1 = _run_ours(x, wt, b, stride, dy)
    y2, dx2, dw2, db2 = _run_ours(x, wt, b, stride, dy)
    assert y1.shape == y64.shape and dw1.dtype == torch.float32 and db1.dtype == torch.float32
    pairs = [("y", y1, yt, y64), ("dW", dw1, wtt.grad, w64.grad), ("db", db1, bt.grad, b64.grad)]
    if need_dx:
        assert dx1.dtype == x.dtype and dx1.shape == x.shape
        pairs.append(("dx", dx1, xt.grad, x64.grad))
    else:
        assert dx1 is None
    for name, ours, torch_bf16, ref in pairs:
        e_ours, e_torch = _rel_rms(ours, ref), _rel_rms(torch_bf16, ref)
        assert e_ours <= RATIO * e_torch, (name, e_ours, e_torch)
    for a, c in ((y1, y2), (dx1, dx2), (dw1, dw2), (db1, db2)):
        assert (a is None and c is None) or torch.equal(a, c)


def test_fp32_output_without_autocast_and_no_bias():
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(3)
    x = torch.randn(1, 64, 3, 16, 16, device=dev, generator=g).requires_grad_(True)
    w = (torch.randn(64, 64, 3, 3, 3, device=dev, generator=g) * 0.03).requires_grad_(True)
    y = VT.causal_conv3d(x, w, None)
    assert y.dtype == torch.float32
    y.backward(torch.ones_like(y))
    assert x.grad.dtype == torch.float32 and w.grad.dtype == torch.float32
    x64, w64 = x.detach().bfloat16().double().requires_grad_(True), w.detach().bfloat16().double().requires_grad_(True)
    y64 = _reference_conv(x64, w64, None, (1, 1, 1))
    y64.backward(torch.ones_like(y64))
    assert _rel_rms(y, y64) < 1e-5 and _rel_rms(x.grad, x64.grad) < 1e-2 and _rel_rms(w.grad, w64.grad) < 1e-5


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("layout", ["contiguous", "channels_last_3d", "sliced"])
@pytest.mark.parametrize("form", ["forward", "gradient_s122", "gradient_s211"])
def test_pack_layouts_and_bias_gradient(dtype, layout, form):
    """pf_conv3d_pack against the same re-layout in torch ops, bit for bit, for the vector (W- or C-contiguous) and the
    scalar loads; the bias gradient against an fp64 sum."""
    from pyramid_flow_b200 import ops
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(7)
    b, c, t, h, w = 2, 72, 3, 10, 48
    src = torch.randn(b, c, t, h, w + 3, device=dev, generator=g).to(dtype)
    src = src[..., :w] if layout == "sliced" else src[..., :w].contiguous()     # sliced: W row stride 51, scalar loads
    if layout == "channels_last_3d":
        src = src.contiguous(memory_format=torch.channels_last_3d)
    dil, t_offset, t_total = {"forward": ((1, 1, 1), 2, t + 2), "gradient_s122": ((1, 2, 2), 0, t + 2),
                              "gradient_s211": ((2, 1, 1), 0, 2 * t + 1)}[form]
    dst = torch.full((b, t_total, h * dil[1], w * dil[2], 128), 7.0, device=dev, dtype=torch.bfloat16)
    db = torch.empty(c, device=dev) if form != "forward" else None
    ops.conv3d_pack(src, dst, t_offset=t_offset, dil=dil, bias_grad=db)
    want = torch.zeros_like(dst)
    want[:, t_offset:t_offset + (t - 1) * dil[0] + 1:dil[0], ::dil[1], ::dil[2], :c] = src.permute(0, 2, 3, 4, 1).bfloat16()
    assert torch.equal(dst, want)
    if db is not None:
        ref = src.double().sum(dim=(0, 2, 3, 4))
        assert (db.double() - ref).abs().max().item() <= 1e-5 * src.double().abs().sum(dim=(0, 2, 3, 4)).max().item()


def test_checkpoint_drops_the_packed_input():
    """Under non-reentrant checkpointing (the reference encoder's mode) the packed input is a saved tensor like any other:
    it is dropped after the forward and recomputed for the backward, so a checkpointed conv holds only its input."""
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(9)
    x = torch.randn(2, 128, 9, 64, 64, device=dev, generator=g).requires_grad_(True)
    w = (torch.randn(128, 128, 3, 3, 3, device=dev, generator=g) * 0.02).requires_grad_(True)
    packed_bytes = 2 * 11 * 64 * 64 * 128 * 2

    def held_after_forward(checkpointed):
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            if checkpointed:
                y = torch.utils.checkpoint.checkpoint(VT.causal_conv3d, x, w, None, use_reentrant=False)
            else:
                y = VT.causal_conv3d(x, w, None)
        torch.cuda.synchronize()
        held = torch.cuda.memory_allocated() - before - y.numel() * y.element_size()
        y.float().sum().backward()
        return held

    plain = held_after_forward(False)
    grads = (x.grad.clone(), w.grad.clone())
    x.grad = w.grad = None
    ckpt = held_after_forward(True)
    assert plain >= packed_bytes, plain
    assert ckpt < packed_bytes // 4, (ckpt, plain)
    assert torch.equal(x.grad, grads[0]) and torch.equal(w.grad, grads[1])


def test_odd_spatial_size_under_spatial_stride_raises():
    x = torch.randn(1, 64, 3, 10, 11, device="cuda")
    with pytest.raises(ValueError, match="even H and W"):
        VT.causal_conv3d(x, torch.randn(64, 64, 3, 3, 3, device="cuda"), None, (1, 2, 2))


# ---- the drop-in on a tiny unmodified reference CausalVideoVAE ------------------------------------------------------------
@pytest.fixture(autouse=True)
def _deterministic_torch(monkeypatch):
    """The torch side of the step with fixed bits and an fp32 reference without TF32: deterministic cuDNN, the math SDPA
    backend for the mid-block attention."""
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
    return vae.cuda().train()


def _step(vae, x, *, autocast: bool, freeze_encoder=False):
    vae.zero_grad(set_to_none=True)
    gen = torch.Generator().manual_seed(5)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        posterior, dec = vae(x, sample_posterior=True, generator=gen, freeze_encoder=freeze_encoder)
        loss = (dec.float() - x).abs().mean() + 1e-3 * posterior.kl().mean()
    loss.backward()
    return loss.detach(), {n: p.grad.detach().clone() for n, p in vae.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("frames", [9, 1])
@pytest.mark.parametrize("checkpointing", [False, True])
@pytest.mark.parametrize("freeze_encoder", [False, True])
def test_tiny_vae_training_step(frames, checkpointing, freeze_encoder):
    if freeze_encoder and checkpointing:
        pytest.skip("freeze_encoder runs the encoder under no_grad: checkpointing changes nothing there")
    vae = _vae()
    for p in list(vae.encoder.parameters()) + list(vae.quant_conv.parameters()):
        p.requires_grad_(not freeze_encoder)
    # the encoder only: the reference decoder hands keyword arguments to a custom_forward(*inputs) under checkpointing
    # (video_vae/modeling_enc_dec.py:313-329), so its own checkpointed forward raises a TypeError with or without the install
    vae.encoder.gradient_checkpointing = checkpointing
    x = torch.randn(2, 3, frames, 32, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(frames))

    fe = dict(freeze_encoder=freeze_encoder)
    loss32, g32 = _step(vae, x, autocast=False, **fe)
    loss_t, g_t = _step(vae, x, autocast=True, **fe)
    VT.install_training_convs(vae)
    try:
        loss_o, g_o = _step(vae, x, autocast=True, **fe)
        loss_o2, g_o2 = _step(vae, x, autocast=True, **fe)
    finally:
        VT.uninstall_training_convs(vae)
    assert set(g_o) == set(g_t) == set(g32)
    if freeze_encoder:
        assert not any(n.startswith(("encoder.", "quant_conv.")) for n in g_o)
    e_loss_o, e_loss_t = abs(loss_o.item() - loss32.item()), abs(loss_t.item() - loss32.item())
    assert e_loss_o <= RATIO * e_loss_t + 1e-4 * abs(loss32.item()), (e_loss_o, e_loss_t)
    worse = []
    for n in g32:
        e_o, e_t = _rel_rms(g_o[n], g32[n]), _rel_rms(g_t[n], g32[n])
        if e_o > RATIO * e_t + 1e-4:
            worse.append((n, e_o, e_t))
    assert not worse, worse
    assert torch.equal(loss_o, loss_o2) and all(torch.equal(g_o[n], g_o2[n]) for n in g_o)


def test_last_layer_grad_then_backward_matches_one_backward():
    """LPIPSWithDiscriminator.calculate_adaptive_weight (video_vae/modeling_loss.py:89-96) takes autograd.grad of the loss
    terms w.r.t. get_last_layer() with retain_graph=True, twice, before the step's backward."""
    vae = _vae(seed=13)
    VT.install_training_convs(vae)
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
        assert g1.shape == last.shape and torch.isfinite(g1).all() and torch.isfinite(g2).all()
        loss.backward()
        again = {n: p.grad for n, p in vae.named_parameters() if p.grad is not None}
    finally:
        VT.uninstall_training_convs(vae)
    assert set(again) == set(plain)
    for n in plain:
        assert torch.equal(again[n], plain[n]), n


def test_uninstall_gives_the_reference_bits_again():
    vae = _vae(seed=17)
    x = torch.randn(1, 3, 5, 32, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    loss_a, g_a = _step(vae, x, autocast=True)
    VT.install_training_convs(vae)
    loss_i, _ = _step(vae, x, autocast=True)
    VT.uninstall_training_convs(vae)
    loss_b, g_b = _step(vae, x, autocast=True)
    assert not torch.equal(loss_i, loss_a)          # the install did run other kernels
    assert torch.equal(loss_a, loss_b) and all(torch.equal(g_a[n], g_b[n]) for n in g_a)
