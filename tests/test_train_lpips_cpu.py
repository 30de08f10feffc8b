"""Training LPIPS of the causal video VAE, host side (no GPU): an fp64 restatement of the distance head's forward and of the
closed-form backward pf_lpips_tap_bwd implements (with a zero feature vector under the ReLU select, and a given dropout
mask) against autograd of the reference's normalize_tensor / lin / spatial_average; the max-pool tie rule against CPU
max_pool2d; what install_training_lpips patches, restores and refuses on the reference LPIPS; and the C-ABI's checks."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from pyramid_flow_b200 import _lib
from pyramid_flow_b200 import vae_training as VT

TAP_CHANNELS = (64, 128, 256, 512, 512)
_FEATURE_SLICES = {1: range(0, 4), 2: range(4, 9), 3: range(9, 16), 4: range(16, 23), 5: range(23, 30)}


def synthetic_lpips_state(seed: int = 0) -> dict:
    """A state_dict for the reference LPIPS: torchvision's VGG16 init (seeded) and non-negative lin weights."""
    from torchvision import models
    with torch.random.fork_rng():
        torch.manual_seed(seed)
        feats = models.vgg16(weights=None).features
    g = torch.Generator().manual_seed(seed + 1)
    sd = {}
    for s, idx in _FEATURE_SLICES.items():
        for i in idx:
            for k, v in feats[i].state_dict().items():
                sd[f"net.slice{s}.{i}.{k}"] = v.clone()
            if isinstance(feats[i], nn.Conv2d):     # VGG's init has zero biases: small ones exercise the bias add
                sd[f"net.slice{s}.{i}.bias"] = 0.05 * torch.randn(feats[i].out_channels, generator=g)
    for k, c in enumerate(TAP_CHANNELS):
        sd[f"lin{k}.model.1.weight"] = torch.rand(1, c, 1, 1, generator=g) * (2.0 / c)
    sd["scaling_layer.shift"] = torch.tensor([-.030, -.088, -.188])[None, :, None, None]
    sd["scaling_layer.scale"] = torch.tensor([.458, .448, .450])[None, :, None, None]
    return sd


def reference_lpips_cls():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    return __import__("video_vae.modeling_lpips", fromlist=["LPIPS"]).LPIPS


def reference_lpips(tmp_path, seed: int = 0):
    path = tmp_path / f"lpips_{seed}.pth"
    torch.save(synthetic_lpips_state(seed), path)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")           # torchvision's `pretrained` deprecation inside the reference
        return reference_lpips_cls()(lpips_ckpt_path=str(path))


# ---- the head's algebra in fp64 ---------------------------------------------------------------------------------------
def _normalize(x, eps=1e-10):
    """normalize_tensor (video_vae/modeling_lpips.py:107-110)."""
    return x / (torch.sqrt(torch.sum(x ** 2, dim=1, keepdim=True)) + eps)


def head_reference(f0, f1, lins, masks, keep_scale):
    """sum_k spatial_average(lin_k(dropout((f0^ - f1^)^2))) of NCHW taps, the dropout given as keep masks."""
    val = 0
    for a, b, w, m in zip(f0, f1, lins, masks):
        d = (_normalize(a) - _normalize(b)) ** 2
        if m is not None:
            d = d * m * keep_scale
        val = val + F.conv2d(d, w.view(1, -1, 1, 1)).mean([2, 3], keepdim=True)
    return val


def tap_backward_closed_form(f, fo, w, m, keep_scale, g, eps=1e-10):
    """pf_lpips_tap_bwd's head gradient of one NCHW tap (no select, no route): a = 2 g / HW * w m (u - uo),
    df = a / (|f| + eps) - f (a . f) / (|f| (|f| + eps)^2), 0 where |f| = 0."""
    hw = f.shape[2] * f.shape[3]
    nrm = torch.sqrt((f * f).sum(1, keepdim=True))
    u, uo = f / (nrm + eps), fo / (torch.sqrt((fo * fo).sum(1, keepdim=True)) + eps)
    scale = w.view(1, -1, 1, 1) * (m * keep_scale if m is not None else 1)
    a = 2 * g.view(-1, 1, 1, 1) / hw * scale * (u - uo)
    dot = (a * f).sum(1, keepdim=True)
    df = a / (nrm + eps) - f * dot / (nrm * (nrm + eps) ** 2)
    return torch.where(nrm > 0, df, torch.zeros_like(df))


@pytest.mark.parametrize("dropout", [False, True])
def test_head_forward_and_closed_form_backward_fp64(dropout):
    g = torch.Generator().manual_seed(3 + dropout)
    n, p = 3, 0.5
    shapes = [(64, 8, 8), (128, 4, 4)]
    f0 = [F.relu(torch.randn(n, c, h, w, generator=g, dtype=torch.float64)) for c, h, w in shapes]
    f1 = [F.relu(torch.randn(n, c, h, w, generator=g, dtype=torch.float64)).requires_grad_(True) for c, h, w in shapes]
    with torch.no_grad():
        f1[0][1, :, 2, 3] = 0                       # a zero feature vector in the branch that takes the gradient
        f0[1][0, :, 1, 1] = 0                       # and one in the other branch
    lins = [torch.rand(c, generator=g, dtype=torch.float64) for c, _, _ in shapes]
    masks = [(torch.rand(n, c, h, w, generator=g) >= p).double() if dropout else None for c, h, w in shapes]
    ks = 1 / (1 - p)
    val = head_reference(f0, f1, lins, masks, ks)
    up = torch.randn(n, 1, 1, 1, generator=g, dtype=torch.float64)
    grads = torch.autograd.grad(val, f1, up)
    # torch's normalize_tensor backward is NaN exactly at the zero vector; the ReLU select (threshold_backward on the
    # result) drops it there, which is what the reference's relu_ does in the full module
    assert torch.isnan(grads[0][1, :, 2, 3]).all()
    for k in range(len(shapes)):
        ours = tap_backward_closed_form(f1[k].detach(), f0[k], lins[k], masks[k], ks, up.view(-1))
        ref = torch.where(f1[k].detach() > 0, grads[k], torch.zeros_like(grads[k]))
        assert torch.isfinite(ours).all()
        torch.testing.assert_close(torch.where(f1[k].detach() > 0, ours, torch.zeros_like(ours)), ref, rtol=1e-9, atol=1e-12)
    # the head is symmetric in its two branches: the other branch's gradient is the same formula with the roles swapped
    f0g = [t.clone().requires_grad_(True) for t in f0]
    g0 = torch.autograd.grad(head_reference(f0g, [t.detach() for t in f1], lins, masks, ks), f0g, up)
    ours0 = tap_backward_closed_form(f0[0], f1[0].detach(), lins[0], masks[0], ks, up.view(-1))
    torch.testing.assert_close(torch.where(f0[0] > 0, ours0, torch.zeros_like(ours0)),
                               torch.where(f0[0] > 0, g0[0], torch.zeros_like(g0[0])), rtol=1e-9, atol=1e-12)


def first_max_route(x, dy):
    """The max-pool backward the kernels implement: dy of each 2x2 window to its first maximum in row-major order."""
    n, c, h, w = x.shape
    win = x.view(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)
    first = win.argmax(-1)                          # torch.argmax returns the first maximal index
    onehot = F.one_hot(first, 4).to(dy.dtype) * dy.unsqueeze(-1)
    return onehot.view(n, c, h // 2, w // 2, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h, w)


def test_maxpool_tie_rule_matches_cpu_max_pool2d():
    g = torch.Generator().manual_seed(5)
    x = torch.randint(0, 3, (2, 8, 6, 10), generator=g).float().requires_grad_(True)   # mostly ties
    y = F.max_pool2d(x, 2, 2)
    dy = torch.randn(y.shape, generator=g)
    y.backward(dy)
    torch.testing.assert_close(first_max_route(x.detach(), dy), x.grad, rtol=0, atol=0)


# ---- the drop-in on the reference LPIPS -------------------------------------------------------------------------------
def _tree(m):
    return [(n, type(s).__name__, id(s)) for n, s in m.named_modules()]


def test_install_and_uninstall_restore_the_module(tmp_path):
    lp = reference_lpips(tmp_path)
    tree, state = _tree(lp), {k: v.clone() for k, v in lp.state_dict().items()}
    VT.install_training_lpips(lp)
    assert lp.forward.__func__ is VT._patched_lpips_forward
    VT.uninstall_training_lpips(lp)
    assert "forward" not in lp.__dict__ and not hasattr(lp, VT._LPIPS_MARK)
    assert _tree(lp) == tree and set(lp.state_dict()) == set(state)
    assert all(torch.equal(lp.state_dict()[k], v) for k, v in state.items())


def test_install_through_the_loss_and_the_wrapper(tmp_path):
    lp = reference_lpips(tmp_path)

    class Loss(nn.Module):                         # LPIPSWithDiscriminator's shape: .perceptual_loss
        def __init__(self):
            super().__init__()
            self.perceptual_loss = lp

    class Wrapper(nn.Module):                      # CausalVideoVAELossWrapper's shape: .loss
        def __init__(self):
            super().__init__()
            self.loss = Loss()

    for owner in (Loss(), Wrapper()):
        VT.install_training_lpips(owner)
        assert lp.forward.__func__ is VT._patched_lpips_forward
        VT.uninstall_training_lpips(owner)
        assert "forward" not in lp.__dict__


def test_lpips_composes_with_the_conv_and_norm_installs(tmp_path):
    from tests.test_train_vae_conv_cpu import TINY_VAE, _reference_vae_cls
    vae = _reference_vae_cls()(**TINY_VAE)
    lp = reference_lpips(tmp_path)

    class Wrapper(nn.Module):
        def __init__(self):
            super().__init__()
            self.vae = vae
            self.loss = nn.Module()
            self.loss.perceptual_loss = lp

    w = Wrapper()
    tree = _tree(w)
    installs = [VT.install_training_lpips, VT.install_training_convs, VT.install_training_norms]
    for order in (installs, installs[::-1]):
        for f in order:
            f(w)
        assert lp.forward.__func__ is VT._patched_lpips_forward
        assert vae.encoder.conv_in.forward.__func__ is VT._patched_forward
        VT.uninstall_training_convs(w)
        VT.uninstall_training_lpips(w)
        VT.uninstall_training_norms(w)
        assert _tree(w) == tree and "forward" not in lp.__dict__


def _set_conv(lp, attr, value, index=2):
    setattr(lp.net.slice1[index], attr, value)


@pytest.mark.parametrize("change, match", [
    (lambda lp: lp.lin2.model[1].weight.requires_grad_(True), "require grad"),
    (lambda lp: setattr(lp.net.slice1[2], "padding", (0, 0)), "pad 1"),
    (lambda lp: setattr(lp.net.slice1[2], "stride", (2, 2)), "stride 1"),
    (lambda lp: setattr(lp.net.slice1[2], "kernel_size", (5, 5)), "3x3"),
    (lambda lp: setattr(lp.net.slice2, "4", nn.MaxPool2d(3, 2)), "MaxPool2d"),
    (lambda lp: setattr(lp.net.slice2, "4", nn.AvgPool2d(2, 2)), "MaxPool2d"),
    (lambda lp: setattr(lp.net.slice3, "11", nn.SiLU()), "nn.ReLU"),
    (lambda lp: lp.net.slice5.add_module("30", nn.MaxPool2d(2, 2)), "slice5"),
    (lambda lp: setattr(lp.lin1, "model", nn.Sequential(nn.Dropout(), nn.Conv2d(128, 1, 1, bias=True)).requires_grad_(False)), "bias-free"),
    (lambda lp: setattr(lp.lin1, "model", nn.Sequential(nn.ReLU(), nn.Conv2d(128, 1, 1, bias=False)).requires_grad_(False)), "bias-free"),
    (lambda lp: setattr(lp.lin1, "model", nn.Sequential(nn.Conv2d(128, 2, 1, bias=False)).requires_grad_(False)), "bias-free"),
    (lambda lp: setattr(lp.lin3.model[0], "p", 1.0), "dropout p=1.0"),
])
def test_install_refusals(tmp_path, change, match):
    lp = reference_lpips(tmp_path)
    change(lp)
    with pytest.raises(ValueError, match=match):
        VT.install_training_lpips(lp)
    assert "forward" not in lp.__dict__


def test_a_lin_layer_without_dropout_is_accepted(tmp_path):
    lp = reference_lpips(tmp_path)
    lp.lin4.model = nn.Sequential(lp.lin4.model[1])
    VT.install_training_lpips(lp)
    VT.uninstall_training_lpips(lp)


def test_install_refuses_what_is_not_lpips():
    with pytest.raises(ValueError, match="no LPIPS"):
        VT.install_training_lpips(nn.Sequential(nn.Conv2d(3, 3, 3)))


def test_op_argument_checks(tmp_path):
    lp = reference_lpips(tmp_path)
    x = torch.randn(2, 3, 32, 32)
    with pytest.raises(ValueError, match="multiples of 16"):
        VT.lpips(torch.randn(2, 3, 32, 40), torch.randn(2, 3, 32, 40), lp)
    with pytest.raises(ValueError, match="one \\[N, 3, H, W\\]"):
        VT.lpips(x, torch.randn(1, 3, 32, 32), lp)
    with pytest.raises(TypeError, match="bf16 or fp32"):
        VT.lpips(x.half(), x.half(), lp)
    with pytest.raises(RuntimeError, match="CPU"):
        VT.lpips(x, x, lp)
    lp2 = copy.deepcopy(lp)
    lp2.lin0.model[0].p = 0.3
    lp2.train()
    with pytest.raises(ValueError, match="different dropout"):
        VT._lpips_dropout(lp2)
    lp.train()
    assert VT._lpips_dropout(lp) == 0.5
    lp.eval()
    assert VT._lpips_dropout(lp) == 0.0


# ---- C-ABI argument checks (no launch happens: every check fails before one) -------------------------------------------
_FAKE = 1 << 20


def _head_desc(**kw):
    d = _lib.LpipsHeadDesc()
    d.n, d.taps = 2, 5
    for k, c in enumerate(TAP_CHANNELS):
        d.f0[k] = d.f1[k] = d.lin[k] = _FAKE
        d.c[k], d.h[k], d.w[k] = c, 64 >> k, 64 >> k
    d.p, d.seed, d.val, d.workspace, d.workspace_floats = 0.0, None, _FAKE, _FAKE, 5 * 2 * _lib.LPIPS_HEAD_BLOCKS
    for k, v in kw.items():
        if k == "c0":
            d.c[0] = v
        elif k == "f1_3":
            d.f1[3] = v
        else:
            setattr(d, k, v)
    return d


@pytest.mark.parametrize("kw, msg", [
    (dict(c0=96), "64, 128, 256 or 512"),
    (dict(taps=6), "taps=6"),
    (dict(n=0), "images"),
    (dict(p=1.0), "dropout p="),
    (dict(p=0.5), "seed"),
    (dict(workspace_floats=10), "too small"),
    (dict(f1_3=None), "null pointer at tap 3"),
    (dict(f1_3=_FAKE + 8), "16-byte aligned"),
    (dict(val=None), "null pointer"),
])
def test_c_abi_refuses_bad_head_descriptors(kw, msg):
    lib = _lib.load()
    assert lib.pf_lpips_head_fwd(C.byref(_head_desc(**kw)), None) != 0
    assert msg in lib.pf_last_error().decode()


def _tap_desc(**kw):
    d = _lib.LpipsTapBwdDesc()
    d.n, d.c, d.h, d.w, d.tap = 2, 64, 16, 16, 0
    d.f = d.f_other = d.lin = d.grad = d.d_next = d.dz = _FAKE
    d.p, d.seed = 0.0, None
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("kw, msg", [
    (dict(c=32), "64, 128, 256 or 512"),
    (dict(h=15), "even h and w"),
    (dict(tap=5), "tap=5"),
    (dict(p=-0.1), "dropout p="),
    (dict(p=0.5), "seed"),
    (dict(grad=None), "null pointer"),
    (dict(dz=_FAKE + 2), "16-byte aligned"),
])
def test_c_abi_refuses_bad_tap_descriptors(kw, msg):
    lib = _lib.load()
    assert lib.pf_lpips_tap_bwd(C.byref(_tap_desc(**kw)), None) != 0
    assert msg in lib.pf_last_error().decode()


def test_c_abi_refuses_bad_pool_and_mask_arguments():
    lib = _lib.load()
    assert lib.pf_maxpool2x2(_FAKE, _FAKE, 2, 15, 16, 64, None) != 0 and "even" in lib.pf_last_error().decode()
    assert lib.pf_maxpool2x2(_FAKE, _FAKE, 2, 16, 16, 12, None) != 0 and "multiple of 8" in lib.pf_last_error().decode()
    assert lib.pf_maxpool2x2(_FAKE + 4, _FAKE, 2, 16, 16, 64, None) != 0 and "aligned" in lib.pf_last_error().decode()
    assert lib.pf_maxpool2x2_bwd(_FAKE, None, _FAKE, 2, 16, 16, 64, None) != 0 and "null" in lib.pf_last_error().decode()
    assert lib.pf_lpips_dropout_mask(_FAKE, 0, 2, 16, 16, 64, 1.5, _FAKE, None) != 0
    assert "dropout p=" in lib.pf_last_error().decode()
    assert lib.pf_lpips_dropout_mask(None, 0, 2, 16, 16, 64, 0.5, _FAKE, None) != 0
    assert "null pointer" in lib.pf_last_error().decode()


def _conv_desc(**kw):
    d = _lib.ConvDesc()
    d.x, d.b, d.t, d.h, d.w, d.cin = _FAKE, 2, 1, 16, 16, 64
    d.wgt, d.cout, d.kt, d.kh, d.kw = _FAKE, 64, 1, 3, 3
    d.out, d.out_t_total, d.out_c, d.store_channels = _FAKE, 1, 64, 64
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("kw, msg", [
    (dict(relu=2), "relu must be 0 or 1"),
    (dict(relu=1, residual=_FAKE), "without a residual"),
    (dict(select=_FAKE, residual=_FAKE), "without a residual"),
    (dict(relu=1, select=_FAKE), "one at a time"),
    (dict(relu=1, store_mode=1, out_c=16), "plain-store"),
    (dict(select=_FAKE, kt=3, store_mode=2, out_c=32), "plain-store"),
    (dict(select=_FAKE, store_channels=32), "store_channels == out_c"),
    (dict(select=_FAKE + 8), "16-byte aligned"),
])
def test_c_abi_refuses_bad_conv_epilogue_fields(kw, msg):
    lib = _lib.load()
    assert lib.pf_causal_conv3d(C.byref(_conv_desc(**kw)), None) != 0
    assert msg in lib.pf_last_error().decode()
