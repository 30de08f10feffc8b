"""Training GroupNorm (+ SiLU) of the causal video VAE, host side (no GPU): an fp64 restatement of the algebra the kernels
implement (pivot-shifted partial sums per (frame, split, channel) -> mean / rstd; backward partials of dz and dz * xhat ->
A, B -> dx, and dgamma / dbeta from the same partials) against autograd of F.group_norm + F.silu on the reference's
rearrange; what install_training_norms patches, swaps, restores and refuses; and the C-ABI's argument checks."""
import ctypes as C

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from pyramid_flow_b200 import _lib, ops
from pyramid_flow_b200 import vae_training as VT
from tests.test_train_vae_conv_cpu import TINY_VAE, _reference_vae_cls


def _reference_norm(x, gamma, beta, groups, eps, silu):
    """CausalGroupNorm.forward (video_vae/modeling_causal_conv.py:36-43), then SiLU."""
    b, c, t, h, w = x.shape
    y = F.group_norm(x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w), groups, gamma, beta, eps)
    y = y.reshape(b, t, c, h, w).permute(0, 2, 1, 3, 4)
    return F.silu(y) if silu else y


def _splits(voxels):
    return min(max((voxels + 4095) // 4096, 1), 64)


def _kernel_algebra(x, dy, gamma, beta, groups, eps, silu, nsplit):
    """The kernels' sums, restated in fp64: x, dy [B, C, T, V]."""
    b, c, t, v = x.shape
    cpg = c // groups
    xf = x.permute(0, 2, 1, 3).reshape(b * t, c, v)                      # [frame, c, voxel]
    dyf = dy.permute(0, 2, 1, 3).reshape(b * t, c, v)
    bounds = [v * s // nsplit for s in range(nsplit + 1)]
    k = xf[:, :, :1]                                                       # the pivot: voxel 0 of each (frame, channel)
    part = torch.stack([torch.stack(((xf[:, :, a:e] - k).sum(-1), ((xf[:, :, a:e] - k) ** 2).sum(-1)), -1)
                        for a, e in zip(bounds[:-1], bounds[1:])], 1)      # [frame, split, c, 2]
    sc, ssc = part[..., 0].sum(1), part[..., 1].sum(1)                     # [frame, c]
    kk = k[..., 0]
    s = (sc + v * kk).view(b * t, groups, cpg).sum(-1)
    ss = (ssc + 2 * kk * sc + v * kk * kk).view(b * t, groups, cpg).sum(-1)
    n = v * cpg
    mean = s / n
    rstd = 1.0 / torch.sqrt((ss / n - mean * mean).clamp_min(0) + eps)
    mean_c = mean.repeat_interleave(cpg, 1)[..., None]
    rstd_c = rstd.repeat_interleave(cpg, 1)[..., None]
    xh = (xf - mean_c) * rstd_c
    z = xh * gamma[None, :, None] + beta[None, :, None]
    act = F.silu(z) if silu else z
    if silu:
        sg = torch.sigmoid(z)
        dz = dyf * sg * (1 + z * (1 - sg))
    else:
        dz = dyf
    bpart = torch.stack([torch.stack((dz[:, :, a:e].sum(-1), (dz[:, :, a:e] * xh[:, :, a:e]).sum(-1)), -1)
                         for a, e in zip(bounds[:-1], bounds[1:])], 1)     # [frame, split, c, 2]
    per_c = bpart.sum(1)                                                   # [frame, c, 2]
    A = (gamma[None] * per_c[..., 0]).view(b * t, groups, cpg).sum(-1) / n
    B = (gamma[None] * per_c[..., 1]).view(b * t, groups, cpg).sum(-1) / n
    dx = rstd_c * (gamma[None, :, None] * dz - A.repeat_interleave(cpg, 1)[..., None] - xh * B.repeat_interleave(cpg, 1)[..., None])
    dbeta = bpart[..., 0].reshape(-1, c).sum(0)
    dgamma = bpart[..., 1].reshape(-1, c).sum(0)
    back = lambda f: f.view(b, t, c, v).permute(0, 2, 1, 3)              # noqa: E731
    return back(act), back(dx), dgamma, dbeta


@pytest.mark.parametrize("t", [1, 3])
@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("hw", [(6, 10), (70, 64)])       # one split; 2 splits of 4480 voxels
def test_backward_algebra_fp64(t, silu, hw):
    g = torch.Generator().manual_seed(t * 7 + silu + hw[0])
    b, c, groups, eps = 2, 16, 4, 1e-6
    h, w = hw
    x = (torch.randn(b, c, t, h, w, generator=g, dtype=torch.float64) * 2 + 3).requires_grad_(True)
    gamma = (1 + 0.3 * torch.randn(c, generator=g, dtype=torch.float64)).requires_grad_(True)
    beta = (0.2 * torch.randn(c, generator=g, dtype=torch.float64)).requires_grad_(True)
    y = _reference_norm(x, gamma, beta, groups, eps, silu)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    dx_ref, dg_ref, db_ref = torch.autograd.grad(y, (x, gamma, beta), dy)
    act, dx, dgamma, dbeta = _kernel_algebra(x.detach().reshape(b, c, t, h * w), dy.reshape(b, c, t, h * w),
                                             gamma.detach(), beta.detach(), groups, eps, silu, _splits(h * w))
    torch.testing.assert_close(act.reshape(y.shape), y.detach(), rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dx.reshape(x.shape), dx_ref, rtol=1e-9, atol=1e-9)
    torch.testing.assert_close(dgamma, dg_ref, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dbeta, db_ref, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("layout, form", [
    (lambda x: x.contiguous(memory_format=torch.channels_last_3d), "channel"),
    (lambda x: x.contiguous(), "plane"),
    (lambda x: x.permute(0, 2, 1, 3, 4).contiguous().permute(0, 2, 1, 3, 4), "plane"),   # [B, T, C, H, W] storage
    (lambda x: x.contiguous()[..., :5], None),                                          # sliced W: neither
    (lambda x: x.permute(0, 1, 2, 4, 3).contiguous().permute(0, 1, 2, 4, 3), None),     # H, W swapped
])
def test_layout_forms(layout, form):
    x = layout(torch.zeros(2, 16, 3, 4, 6))
    assert ops.groupnorm_form(x) == form


# ---- the drop-in on an unmodified reference CausalVideoVAE --------------------------------------------------------------
def _tiny_vae():
    return _reference_vae_cls()(**TINY_VAE)


def _tree(m):
    return [(n, type(s).__name__, id(s)) for n, s in m.named_modules()]


def test_install_patches_every_group_norm_and_uninstall_restores():
    vae = _tiny_vae()
    norms = VT.causal_group_norms(vae)
    names = {n for n, _ in norms}
    assert {"encoder.conv_norm_out", "decoder.conv_norm_out", "encoder.down_blocks.0.resnets.0.norm1",
            "decoder.mid_block.resnets.0.norm2"} <= names
    tree, state = _tree(vae), {k: v.clone() for k, v in vae.state_dict().items()}
    before = {n: m.forward for n, m in vae.named_modules()}
    VT.install_training_norms(vae)
    for n, m in vae.named_modules():
        if n in names:
            assert m.forward.__func__ is VT._patched_norm_forward, n
        elif type(m).__name__ == "CausalResnetBlock3D":
            assert type(m.nonlinearity) is nn.Identity, n
    assert type(vae.encoder.conv_act) is nn.Identity and type(vae.decoder.conv_act) is nn.Identity
    assert not any(type(m) is nn.SiLU for _, m in vae.named_modules())
    assert set(vae.state_dict()) == set(state)
    VT.install_training_norms(vae)          # a second install changes nothing
    VT.uninstall_training_norms(vae)
    assert _tree(vae) == tree
    assert all(torch.equal(vae.state_dict()[k], v) for k, v in state.items()) and set(vae.state_dict()) == set(state)
    for n, m in vae.named_modules():
        assert "forward" not in m.__dict__ and m.forward == before[n], n
        assert not hasattr(m, VT._NORM_MARK) and VT._SAVED_ACT not in m.__dict__


def test_norms_and_convs_compose_in_either_order():
    vae = _tiny_vae()
    tree = _tree(vae)
    for first, second in ((VT.install_training_norms, VT.install_training_convs),
                          (VT.install_training_convs, VT.install_training_norms)):
        first(vae)
        second(vae)
        assert vae.encoder.conv_in.forward.__func__ is VT._patched_forward
        assert vae.encoder.conv_norm_out.forward.__func__ is VT._patched_norm_forward
        VT.uninstall_training_convs(vae)
        VT.uninstall_training_norms(vae)
        assert _tree(vae) == tree


def test_install_through_the_loss_wrapper_patches_its_vae():
    vae = _tiny_vae()

    class Wrapper(nn.Module):
        def __init__(self, v):
            super().__init__()
            self.vae = v

    wrapper = Wrapper(vae)
    VT.install_training_norms(wrapper)
    assert vae.decoder.conv_norm_out.forward.__func__ is VT._patched_norm_forward
    VT.uninstall_training_norms(wrapper)
    assert "forward" not in vae.decoder.conv_norm_out.__dict__ and type(vae.decoder.conv_act) is nn.SiLU


def _first_resnet(vae):
    return vae.encoder.down_blocks[0].resnets[0]


@pytest.mark.parametrize("change, match", [
    (lambda v: setattr(_first_resnet(v), "nonlinearity", nn.GELU()), "not nn.SiLU"),
    (lambda v: setattr(v.decoder, "conv_act", nn.Mish()), "not nn.SiLU"),
    (lambda v: setattr(_first_resnet(v).dropout, "p", 0.1), "dropout"),
    (lambda v: setattr(_first_resnet(v), "time_embedding_norm", "scale_shift"), "time_embedding_norm"),
    (lambda v: setattr(_first_resnet(v).norm1, "num_channels", 60), "multiple of 8"),
])
def test_install_refusals(change, match):
    vae = _tiny_vae()
    change(vae)
    tree = _tree(vae)
    with pytest.raises(ValueError, match=match):
        VT.install_training_norms(vae)
    assert _tree(vae) == tree                                               # nothing half-installed
    assert all("forward" not in m.__dict__ for _, m in VT.causal_group_norms(vae))


def test_install_refuses_a_model_without_causal_group_norms():
    with pytest.raises(ValueError, match="CausalGroupNorm"):
        VT.install_training_norms(nn.Sequential(nn.GroupNorm(2, 8)))


def test_fp16_and_cpu_tensors_raise():
    x = torch.randn(1, 16, 2, 4, 4)
    w, b = torch.ones(16), torch.zeros(16)
    with pytest.raises(TypeError, match="bf16 or fp32"):
        VT.causal_group_norm(x.half(), w, b, 4, 1e-6)
    with pytest.raises(RuntimeError, match="CPU"):
        VT.causal_group_norm(x, w, b, 4, 1e-6, silu=True)
    with pytest.raises(ValueError, match="multiple of 8"):
        VT.causal_group_norm(torch.randn(1, 12, 2, 4, 4), torch.ones(12), torch.zeros(12), 4, 1e-6)
    vae = _tiny_vae()
    VT.install_training_norms(vae)
    with pytest.raises(RuntimeError, match="CPU"):
        vae.encoder.conv_norm_out(torch.randn(1, 128, 1, 4, 4))


# ---- C-ABI argument checks (no launch happens: every check fails before one) ------------------------------------------
_FAKE = 1 << 20          # a 16-byte aligned address that is never dereferenced


def _desc(**kw):
    d = _lib.GroupNormTrainDesc()
    d.x, d.x_f32, d.b, d.c, d.t, d.h, d.w = _FAKE, 0, 2, 64, 3, 8, 8
    for i, s in enumerate((64 * 3 * 64, 1, 64 * 64, 8 * 64, 64)):            # channels_last_3d
        d.x_strides[i] = s
    d.groups, d.eps, d.silu = 32, 1e-6, 1
    d.gamma = d.beta = d.stats = d.y = d.dy = d.dx = _FAKE
    for i in range(5):
        d.dy_strides[i] = d.x_strides[i]
    for k, v in kw.items():
        if k in ("x_strides", "dy_strides"):
            for i, s in enumerate(v):
                getattr(d, k)[i] = s
        else:
            setattr(d, k, v)
    return d


def test_workspace_query():
    lib = _lib.load()
    d = _desc()
    assert lib.pf_groupnorm_train_workspace(C.byref(d)) == 2 * 3 * 1 * 64 * 2 + 2 * 3 * 32 * 2
    d = _desc(h=128, w=100, x_strides=(64 * 3 * 12800, 1, 64 * 12800, 100 * 64, 64))    # 12800 voxels: 4 splits
    assert lib.pf_groupnorm_train_workspace(C.byref(d)) == 2 * 3 * 4 * 64 * 2 + 2 * 3 * 32 * 2


@pytest.mark.parametrize("kw, msg", [
    (dict(c=60, groups=30, x_strides=(60 * 3 * 64, 1, 60 * 64, 8 * 60, 60)), "multiple of 8"),
    (dict(groups=24), "multiple of groups"),
    (dict(groups=0), "multiple of groups"),
    (dict(h=0), "bad shape"),
    (dict(x_f32=2), "x_f32"),
    (dict(x_strides=(64 * 3 * 64, 1, 64 * 64, 64, 8 * 64)), "neither channels_last_3d nor"),
    (dict(x_strides=(64 * 3 * 80, 3 * 80, 80, 10, 1)), "neither channels_last_3d nor"),
])
def test_c_abi_refuses_bad_descriptors(kw, msg):
    lib = _lib.load()
    d = _desc(**kw)
    assert lib.pf_groupnorm_train_workspace(C.byref(d)) < 0
    assert msg in lib.pf_last_error().decode()
    assert lib.pf_groupnorm_train_fwd(C.byref(d), None) != 0
    assert msg in lib.pf_last_error().decode()


def test_c_abi_refuses_null_pointers_small_workspace_and_a_dy_in_another_form():
    lib = _lib.load()
    d = _desc(workspace=_FAKE, workspace_floats=1 << 20, x=None)
    assert lib.pf_groupnorm_train_fwd(C.byref(d), None) != 0 and "null pointer" in lib.pf_last_error().decode()
    d = _desc(workspace=_FAKE, workspace_floats=1 << 20, dy=None)
    assert lib.pf_groupnorm_train_bwd(C.byref(d), None) != 0 and "null pointer" in lib.pf_last_error().decode()
    d = _desc(workspace=_FAKE, workspace_floats=10)
    assert lib.pf_groupnorm_train_fwd(C.byref(d), None) != 0 and "too small" in lib.pf_last_error().decode()
    d = _desc()
    assert lib.pf_groupnorm_train_fwd(C.byref(d), None) != 0 and "workspace" in lib.pf_last_error().decode()
    d = _desc(workspace=_FAKE, workspace_floats=1 << 20, dy_strides=(64 * 3 * 64, 3 * 64, 64, 8, 1))    # NCDHW dy
    assert lib.pf_groupnorm_train_bwd(C.byref(d), None) != 0 and "layout form" in lib.pf_last_error().decode()
