"""Training LPIPS on the GPU: the VGG convs in their (1, 3, 3) form with the relu / select epilogues, the max-pool bit for
bit against torch, the head and the tap backward against fp64, the whole op's value and input gradient against the
reference LPIPS in fp64 (within 1.5x of torch's bf16 autocast error, in eval mode and with the training dropout given as
the kernels' mask), its repeatability, what it saves and its dropout statistics, and one step of a tiny reference VAE with
the real LPIPSWithDiscriminator."""
import copy
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from pyramid_flow_b200 import ops
from pyramid_flow_b200 import vae_training as VT
from tests.test_train_lpips_cpu import TAP_CHANNELS, head_reference, reference_lpips, synthetic_lpips_state

pytestmark = pytest.mark.gpu

RATIO = 1.5
DEV = torch.device("cuda")


def _rel_rms(a, ref):
    a, ref = a.double(), ref.double()
    return ((a - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt().clamp_min(1e-30)).item()


@pytest.fixture(autouse=True)
def _fp32_reference(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    yield


def _cl(x):        # NCHW -> the kernels' [N, 1, H, W, C]
    return x.permute(0, 2, 3, 1).contiguous().unsqueeze(1)


# ---- the conv kernel in the VGG form ----------------------------------------------------------------------------------
VGG_LAYERS = sorted({(cin, cout, 256 >> s) for s, convs in enumerate(((0, 1), (2, 3), (4, 5, 6), (7, 8, 9), (10, 11, 12)))
                     for cin, cout in (VT.VGG16_CONVS[i] for i in convs)})


@pytest.mark.parametrize("layer", VGG_LAYERS, ids=lambda l: f"{l[0]}to{l[1]}_{l[2]}")
def test_vgg_conv_relu_forward_and_select_data_gradient(layer):
    cin, cout, hw = layer
    n = 2
    g = torch.Generator(device=DEV).manual_seed(cin + cout + hw)
    x = F.relu(torch.randn(n, cin, hw, hw, device=DEV, generator=g)).bfloat16()
    w = (torch.randn(cout, cin, 3, 3, device=DEV, generator=g) * (2.0 / (9 * cin)) ** 0.5).bfloat16()
    b = torch.randn(cout, device=DEV, generator=g) * 0.1
    # forward with the ReLU epilogue
    xp = torch.zeros(n, 1, hw, hw, VT._pad64(cin), device=DEV, dtype=torch.bfloat16)
    xp[..., :cin] = _cl(x)[..., :cin]
    y = torch.empty(n, 1, hw, hw, cout, device=DEV, dtype=torch.bfloat16)
    ops.causal_conv3d(xp, VT._vgg_filter(w), b.contiguous(), y, kernel=(1, 3, 3), relu=True)
    y64 = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        yt = F.relu(F.conv2d(x.float(), w.float(), b, padding=1))
    ours = y[:, 0].permute(0, 3, 1, 2)
    assert (ours >= 0).all()
    assert _rel_rms(ours, y64) <= RATIO * _rel_rms(yt, y64), (_rel_rms(ours, y64), _rel_rms(yt, y64))
    # data gradient, with the ReLU select of the layer in front (x is that layer's ReLU output) where cin is a feature map
    dy = torch.randn(n, cout, hw, hw, device=DEV, generator=g).bfloat16()
    dx64 = F.conv_transpose2d(dy.double(), w.double(), padding=1)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        dxt = F.conv_transpose2d(dy.float(), w.float(), padding=1)
    if cin == 3:
        out = torch.empty(n, 1, hw, hw, 3, device=DEV, dtype=torch.float32)
        ops.causal_conv3d(_cl(dy), VT._vgg_dgrad_filter(w), None, out, kernel=(1, 3, 3), store_channels=3)
    else:
        dx64 = torch.where(x > 0, dx64, torch.zeros_like(dx64))
        dxt = torch.where(x > 0, dxt.float(), torch.zeros_like(dxt.float()))
        out = torch.empty(n, 1, hw, hw, cin, device=DEV, dtype=torch.bfloat16)
        ops.causal_conv3d(_cl(dy), VT._vgg_dgrad_filter(w), None, out, kernel=(1, 3, 3), select=_cl(x))
        assert (out[:, 0].permute(0, 3, 1, 2)[x <= 0] == 0).all()
    dx = out[:, 0].permute(0, 3, 1, 2)
    assert _rel_rms(dx, dx64) <= RATIO * _rel_rms(dxt, dx64), (_rel_rms(dx, dx64), _rel_rms(dxt, dx64))


def test_select_drops_non_finite_gradients():
    n, c, hw = 1, 64, 16
    dy = torch.full((n, 1, hw, hw, c), float("nan"), device=DEV, dtype=torch.bfloat16)
    sel = torch.zeros(n, 1, hw, hw, c, device=DEV, dtype=torch.bfloat16)
    sel[..., 5] = 1
    out = torch.empty_like(sel)
    w = torch.randn(c, c, 3, 3, device=DEV) * 0.05
    ops.causal_conv3d(dy, VT._vgg_dgrad_filter(w), None, out, kernel=(1, 3, 3), select=sel)
    assert (out[..., :5] == 0).all() and (out[..., 6:] == 0).all() and torch.isnan(out[..., 5]).all()


# ---- the max-pool -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(3, 64, 32, 48), (2, 512, 16, 16), (1, 8, 2, 2)])
def test_maxpool_bitwise_against_torch(shape):
    n, c, h, w = shape
    g = torch.Generator(device=DEV).manual_seed(c + h)
    x = (torch.randint(-2, 3, shape, device=DEV, generator=g).float() * 0.25).bfloat16()     # mostly ties
    x[0, 0, 0, 0] = -0.0
    xt = x.clone().requires_grad_(True)
    yt = F.max_pool2d(xt, 2, 2)
    dy = torch.randn(yt.shape, device=DEV, generator=g).bfloat16()
    yt.backward(dy)
    xc = x.permute(0, 2, 3, 1).contiguous()
    y = torch.empty(n, h // 2, w // 2, c, device=DEV, dtype=torch.bfloat16)
    ops.maxpool2x2(xc, y)
    assert torch.equal(y.permute(0, 3, 1, 2).view(torch.int16), yt.detach().view(torch.int16))
    dx = torch.empty_like(xc)
    ops.maxpool2x2_bwd(xc, dy.permute(0, 2, 3, 1).contiguous(), dx)
    assert torch.equal(dx.permute(0, 3, 1, 2), xt.grad)


# ---- the head and the tap backward -------------------------------------------------------------------------------------
def _taps(n, hw, seed, zero_pixels=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for k, c in enumerate(TAP_CHANNELS):
        s = hw >> k
        t = F.relu(torch.randn(n, s, s, c, device=DEV, generator=g) + 0.3).bfloat16()
        if zero_pixels:
            t[:, ::3, ::2] = 0
        out.append(t)
    return out


def _masks(seed, n, hw, p):
    ms = []
    for k, c in enumerate(TAP_CHANNELS):
        m = torch.empty(n, hw >> k, hw >> k, c, device=DEV, dtype=torch.uint8)
        ops.lpips_dropout_mask(seed, m, tap=k, p=p)
        ms.append(m)
    return ms


@pytest.mark.parametrize("p", [0.0, 0.5])
def test_head_and_tap_backward_against_fp64(p):
    n, hw = 3, 32
    f0, f1 = _taps(n, hw, 1), _taps(n, hw, 2, zero_pixels=True)
    g = torch.Generator(device=DEV).manual_seed(3)
    lins = [torch.rand(c, device=DEV, generator=g) * (2.0 / c) for c in TAP_CHANNELS]
    seed = torch.tensor([0x1234_5678_9ABC_DEF], device=DEV, dtype=torch.int64) if p else None
    masks = _masks(seed, n, hw, p) if p else [None] * 5
    val = torch.empty(n, device=DEV)
    ops.lpips_head_fwd(f0, f1, lins, val, p=p, seed=seed)
    nchw = lambda t: t.permute(0, 3, 1, 2).double()                                  # noqa: E731
    f1_64 = [nchw(t).requires_grad_(True) for t in f1]
    ks = 1 / (1 - p)
    ref = head_reference([nchw(t) for t in f0], f1_64, [w.double() for w in lins],
                         [nchw(m) if m is not None else None for m in masks], ks).view(-1)
    assert _rel_rms(val, ref) < 1e-5, (val, ref)
    up = torch.randn(n, device=DEV, generator=g)
    grads = torch.autograd.grad(ref, f1_64, up.double())
    for k in range(5):
        f = f1[k]
        d_next = None
        route = torch.zeros_like(grads[k])
        if k < 4:
            s = f.shape[1]
            d_next = torch.randn(n, s // 2, s // 2, f.shape[3], device=DEV, generator=g).bfloat16()
            xk = nchw(f).requires_grad_(True)
            F.max_pool2d(xk, 2, 2).backward(nchw(d_next))
            route = xk.grad
        want = torch.where(nchw(f) > 0, torch.nan_to_num(grads[k], nan=0.0) + route, torch.zeros_like(route))
        dz = torch.empty_like(f)
        ops.lpips_tap_bwd(f, f0[k], lins[k], up, d_next, dz, tap=k, p=p, seed=seed)
        got = nchw(dz)
        assert torch.isfinite(got).all()
        assert (got[nchw(f) <= 0] == 0).all()
        # one bf16 rounding of the fp32 sum
        assert (got - want).abs().max().item() <= 2 ** -8 * want.abs().max().item() + 1e-12, k
        assert _rel_rms(got, want) < 4e-3, k


def test_dropout_statistics():
    n, hw, p = 2, 64, 0.5
    s1 = torch.tensor([11], device=DEV, dtype=torch.int64)
    s2 = torch.tensor([12], device=DEV, dtype=torch.int64)
    m1, m2 = _masks(s1, n, hw, p), _masks(s2, n, hw, p)
    for k in range(5):
        cnt = m1[k].numel()
        kept = m1[k].sum().item()
        assert abs(kept - cnt * (1 - p)) <= 5 * math.sqrt(cnt * p * (1 - p)), (k, kept, cnt)
        assert not torch.equal(m1[k], m2[k])
    assert not torch.equal(m1[3], m1[4])                                   # same shape, different taps
    m = torch.empty(1, 32, 32, 64, device=DEV, dtype=torch.uint8)
    ops.lpips_dropout_mask(s1, m, tap=0, p=0.2)
    assert abs(m.float().mean().item() - 0.8) < 5 * math.sqrt(0.16 / m.numel())
    again = _masks(s1, n, hw, p)
    assert all(torch.equal(a, b) for a, b in zip(m1, again))


# ---- the whole op ------------------------------------------------------------------------------------------------------
class _MaskedDropout(nn.Module):
    def __init__(self, mask, p):
        super().__init__()
        self.mask, self.scale = mask, 1.0 / (1.0 - p)

    def forward(self, x):
        return x * self.mask.to(x.dtype) * self.scale


def _inputs(n, hw, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x0 = torch.rand(n, 3, hw, hw, device=DEV, generator=g) * 2 - 1
    x1 = (x0 + 0.3 * torch.randn(n, 3, hw, hw, device=DEV, generator=g)).clamp(-1, 1)
    return x0.to(dtype), x1.to(dtype)


def _drawn_seed(torch_seed):
    torch.manual_seed(torch_seed)
    return torch.empty(1, device=DEV, dtype=torch.int64).random_()


@pytest.fixture(scope="module")
def lpips_module(tmp_path_factory):
    return reference_lpips(tmp_path_factory.mktemp("lpips")).cuda()


@pytest.mark.parametrize("n", [1, 34])
@pytest.mark.parametrize("hw", [64, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("mode", ["eval", "train"])
def test_lpips_against_fp64(lpips_module, mode, dtype, hw, n):
    lp = lpips_module.train(mode == "train")
    x0, x1 = _inputs(n, hw, dtype, seed=n + hw)
    up = torch.rand(n, 1, 1, 1, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7)) + 0.5
    torch.manual_seed(1234)
    x1o = x1.clone().requires_grad_(True)
    val = VT.lpips(x0, x1o, lp)
    val.backward(up)
    assert val.shape == (n, 1, 1, 1) and val.dtype == torch.float32 and x1o.grad.dtype == dtype

    ref = copy.deepcopy(lp).double()
    if mode == "train":
        masks = _masks(_drawn_seed(1234), n, hw, 0.5)
        for k, m in enumerate(masks):
            getattr(ref, f"lin{k}").model[0] = _MaskedDropout(m.permute(0, 3, 1, 2), 0.5)
    tref = copy.deepcopy(ref).float()
    x1r = x1.double().requires_grad_(True)
    v64 = ref(x0.double(), x1r)
    v64.backward(up.double())
    x1t = x1.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        vt = tref(x0, x1t)
    vt.float().backward(up)
    e_val, e_val_t = _rel_rms(val, v64), _rel_rms(vt, v64)
    e_dx, e_dx_t = _rel_rms(x1o.grad, x1r.grad), _rel_rms(x1t.grad, x1r.grad)
    assert e_val <= RATIO * e_val_t + 1e-6, (e_val, e_val_t)
    assert e_dx <= RATIO * e_dx_t, (e_dx, e_dx_t)


def test_gradients_to_both_inputs_repeat_bitwise_and_survive_retain_graph(lpips_module):
    lp = lpips_module.train()
    x0, x1 = _inputs(4, 64, torch.float32, seed=5)

    def run():
        torch.manual_seed(99)
        a, b = x0.clone().requires_grad_(True), x1.bfloat16().requires_grad_(True)
        v = VT.lpips(a, b, lp)
        return v, a, b

    v1, a1, b1 = run()
    g_first = torch.autograd.grad(v1.sum(), (a1, b1), retain_graph=True)
    g_second = torch.autograd.grad(v1.sum(), (a1, b1), retain_graph=True)
    v1.sum().backward()
    v2, a2, b2 = run()
    v2.sum().backward()
    assert torch.equal(v1, v2)
    assert b1.grad.dtype == torch.bfloat16 and a1.grad.dtype == torch.float32 and a1.grad.shape == x0.shape
    for x, y in zip(g_first, g_second):
        assert torch.equal(x, y)
    assert torch.equal(a1.grad, a2.grad) and torch.equal(b1.grad, b2.grad) and torch.equal(a1.grad, g_first[0])
    torch.manual_seed(100)
    assert not torch.equal(VT.lpips(x0, x1, lp), v1)                    # a new call draws a new dropout mask
    lp.eval()
    assert torch.equal(VT.lpips(x0, x1, lp), VT.lpips(x0, x1, lp))


def test_what_is_saved(lpips_module):
    lp = lpips_module.eval()
    x0, x1 = _inputs(2, 64, torch.float32, seed=6)
    seen = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: seen.append(tuple(t.shape)) or t, lambda t: t):
        VT.lpips(x0, x1.requires_grad_(True), lp)
    relu_shapes = []
    hw = 64
    for s, nconv in enumerate(VT.VGG16_SLICES):
        hw = hw if s == 0 else hw // 2
        relu_shapes += [(2, 1, hw, hw, TAP_CHANNELS[s])] * nconv
    tap_shapes = [(2, 1, 64 >> s, 64 >> s, c) for s, c in enumerate(TAP_CHANNELS)]
    assert seen == tap_shapes + relu_shapes                           # input branch: its taps; target branch: every ReLU


def test_zero_feature_vectors_give_the_reference_gradient(tmp_path):
    """conv1_2 with 64 identical filters: relu1_2's feature vector is all zero at about half the pixels.  torch's
    normalize_tensor backward is NaN there and its ReLU backward drops it; the op must give the same finite gradient."""
    lp = reference_lpips(tmp_path, seed=3).cuda().eval()
    with torch.no_grad():
        conv = lp.net.slice1[2]
        conv.weight.copy_(conv.weight[:1].expand_as(conv.weight))
        conv.bias.copy_(conv.bias[:1].expand_as(conv.bias))
    x0, x1 = _inputs(2, 32, torch.float32, seed=8)
    x1o = x1.clone().requires_grad_(True)
    VT.lpips(x0, x1o, lp).sum().backward()
    ref = copy.deepcopy(lp).double()
    x1r = x1.double().requires_grad_(True)
    feats = ref.net(ref.scaling_layer(x1r))[0]
    zero_frac = (feats.abs().sum(1) == 0).double().mean().item()
    assert 0.2 < zero_frac < 0.8, zero_frac
    ref(x0.double(), x1r).sum().backward()
    assert torch.isfinite(x1r.grad).all() and torch.isfinite(x1o.grad).all()
    tref = copy.deepcopy(lp)
    x1t = x1.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        tref(x0, x1t).float().sum().backward()
    assert _rel_rms(x1o.grad, x1r.grad) <= RATIO * _rel_rms(x1t.grad, x1r.grad)


# ---- one step of the tiny reference VAE with the real LPIPSWithDiscriminator ---------------------------------------------
def test_tiny_vae_training_step_with_lpips(tmp_path):
    from oracle.pin import ref_shim
    from tests.test_train_vae_conv_cpu import TINY_VAE, _reference_vae_cls
    from torch.nn.attention import SDPBackend, sdpa_kernel
    vae_cls = _reference_vae_cls()
    loss_cls = __import__("video_vae.modeling_loss", fromlist=["LPIPSWithDiscriminator"]).LPIPSWithDiscriminator
    path = tmp_path / "lpips.pth"
    torch.save(synthetic_lpips_state(0), path)
    vae = vae_cls(**TINY_VAE)
    ref_shim.reinit_all_parameters(vae, seed=11, std=0.05)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        loss_mod = loss_cls(disc_start=250000, kl_weight=1e-12, pixelloss_weight=10.0, perceptual_weight=1.0,
                            lpips_ckpt=str(path))

    class Step(nn.Module):
        def __init__(self):
            super().__init__()
            self.vae, self.loss = vae, loss_mod

    model = Step().cuda().train()
    # LPIPS's dropout draws different masks in torch and in the op: the comparison runs LPIPS in eval mode (the dropout
    # itself is checked against the op's own mask above)
    loss_mod.perceptual_loss.eval()
    gen = torch.Generator(device=DEV).manual_seed(21)
    clips = [torch.rand(2, 3, 5, 32, 32, device=DEV, generator=gen) * 2 - 1,
             torch.rand(2, 3, 1, 32, 32, device=DEV, generator=gen) * 2 - 1]

    def step(x, autocast):
        model.zero_grad(set_to_none=True)
        with sdpa_kernel(SDPBackend.MATH), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            posterior, dec = vae(x, sample_posterior=True, generator=torch.Generator().manual_seed(5))
            loss, _ = loss_mod(x, dec, posterior, optimizer_idx=0, global_step=0, last_layer=vae.get_last_layer())
        loss.backward()
        return loss.detach(), {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    for x in clips:
        loss32, g32 = step(x, False)
        loss_t, g_t = step(x, True)
        for f in (VT.install_training_convs, VT.install_training_norms, VT.install_training_lpips):
            f(model)
        try:
            loss_o, g_o = step(x, True)
        finally:
            VT.uninstall_training_lpips(model)
            VT.uninstall_training_norms(model)
            VT.uninstall_training_convs(model)
        assert set(g_o) == set(g_t) == set(g32) and "loss.logvar" in g_o
        e_o, e_t = abs(loss_o.item() - loss32.item()), abs(loss_t.item() - loss32.item())
        assert e_o <= RATIO * e_t + 1e-4 * abs(loss32.item()), (e_o, e_t)
        worse = [(n, _rel_rms(g_o[n], g32[n]), _rel_rms(g_t[n], g32[n])) for n in g32
                 if _rel_rms(g_o[n], g32[n]) > RATIO * _rel_rms(g_t[n], g32[n]) + 1e-4]
        assert not worse, worse
