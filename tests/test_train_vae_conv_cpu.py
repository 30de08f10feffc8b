"""Training convolutions of the causal video VAE, host side (no GPU): the fp64 identities the backward kernels implement
(data gradient = the forward conv on dilated, end-padded dy with the flipped, transposed filter; weight gradient = a sum
of dy x shifted x over the voxels), and what install_training_convs patches, restores and refuses."""
import pytest
import torch
import torch.nn.functional as F

from pyramid_flow_b200 import vae_training as VT

STRIDES = [(1, 1, 1), (1, 2, 2), (2, 1, 1)]


def _reference_conv(x, w, b, stride):
    """CausalConv3d.forward, temporal_chunk=False (video_vae/modeling_causal_conv.py:116-126)."""
    pad = (1, 1, 1, 1, 2, 0) if w.shape[2] == 3 else (0,) * 6
    return F.conv3d(F.pad(x, pad), w, b, stride=stride)


def _dgrad_as_forward_conv(dy, w, x_shape, stride):
    """dx = conv3d(dilate(dy) with kt-1 zero frames at the end, flip(W)^T), spatial pad 1: the forward's own form."""
    _, _, t, h, wd = x_shape
    kt = w.shape[2]
    st, sh, sw = stride
    up = dy.new_zeros(dy.shape[0], dy.shape[1], t + kt - 1, h, wd)
    up[:, :, 0:(dy.shape[2] - 1) * st + 1:st, ::sh, ::sw] = dy
    wb = w.flip(2, 3, 4).transpose(0, 1)
    return F.conv3d(F.pad(up, (1, 1, 1, 1, 0, 0)) if kt == 3 else up, wb)


def _wgrad_as_voxel_sum(dy, x, w_shape, stride):
    """dW[co, ci, tap] = sum over output voxels of dy[v, co] * x_pad[v * stride + tap, ci]."""
    kt, kh, kw = w_shape[2:]
    st, sh, sw = stride
    pad = (1, 1, 1, 1, 2, 0) if kt == 3 else (0,) * 6
    xp = F.pad(x, pad)
    to, ho, wo = dy.shape[2:]
    dw = dy.new_zeros(w_shape)
    for dt in range(kt):
        for dh in range(kh):
            for dwi in range(kw):
                xs = xp[:, :, dt:dt + (to - 1) * st + 1:st, dh:dh + (ho - 1) * sh + 1:sh, dwi:dwi + (wo - 1) * sw + 1:sw]
                dw[:, :, dt, dh, dwi] = torch.einsum("bcthw,bdthw->cd", dy, xs)
    return dw


@pytest.mark.parametrize("stride", STRIDES)
@pytest.mark.parametrize("t", [1, 5, 4])
@pytest.mark.parametrize("k", [3, 1])
def test_backward_identities_fp64(stride, t, k):
    if k == 1 and stride != (1, 1, 1):
        pytest.skip("1x1x1 convs have unit stride")
    g = torch.Generator().manual_seed(t * 10 + stride[0] + 3 * stride[1] + k)
    cin, cout, h, w = 3, 5, 6, 8
    x = torch.randn(2, cin, t, h, w, generator=g, dtype=torch.float64, requires_grad=True)
    wt = torch.randn(cout, cin, k, k, k, generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(cout, generator=g, dtype=torch.float64, requires_grad=True)
    y = _reference_conv(x, wt, b, stride)
    assert tuple(y.shape[2:]) == VT._out_dims(x.shape, stride)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    dx_ref, dw_ref, db_ref = torch.autograd.grad(y, (x, wt, b), dy)

    dx = _dgrad_as_forward_conv(dy, wt.detach(), x.shape, stride)
    assert dx.shape == x.shape
    torch.testing.assert_close(dx, dx_ref, rtol=1e-12, atol=1e-12)
    # the same gradient as conv_transpose3d of the padded input, cropped to x
    kt = wt.shape[2]
    padded = (t + (kt - 1), h + (k - 1), w + (k - 1))
    natural = tuple((n - 1) * s + k for n, s in zip(y.shape[2:], stride))
    gpad = F.conv_transpose3d(dy, wt.detach(), stride=stride, output_padding=tuple(p - q for p, q in zip(padded, natural)))
    if k == 3:
        gpad = gpad[:, :, 2:, 1:-1, 1:-1]
    torch.testing.assert_close(gpad, dx_ref, rtol=1e-12, atol=1e-12)

    torch.testing.assert_close(_wgrad_as_voxel_sum(dy, x.detach(), wt.shape, stride), dw_ref, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dy.sum(dim=(0, 2, 3, 4)), db_ref, rtol=1e-12, atol=1e-12)


def test_filter_layouts():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(5, 3, 3, 3, 3, generator=g)
    wf = VT.forward_filter(w, 64, 64).view(64, 3, 3, 3, 64)
    assert torch.equal(wf[:5, 1, 2, 0, :3], w[:, :, 1, 2, 0].bfloat16())
    assert wf[5:].abs().sum() == 0 and wf[:, ..., 3:].abs().sum() == 0
    wb = VT.dgrad_filter(w, 64, 64).view(64, 3, 3, 3, 64)
    assert torch.equal(wb[:3, 0, 1, 2, :5], w[:, :, 2, 1, 0].t().bfloat16())


# ---- the drop-in on an unmodified reference CausalVideoVAE --------------------------------------------------------------
def _reference_vae_cls():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    return __import__("video_vae", fromlist=["CausalVideoVAE"]).CausalVideoVAE


TINY_VAE = dict(encoder_in_channels=3, encoder_out_channels=4, decoder_in_channels=4, decoder_out_channels=3,
                encoder_layers_per_block=(1, 1), encoder_down_block_types=("DownEncoderBlockCausal3D",) * 2,
                encoder_block_out_channels=(64, 128), encoder_spatial_down_sample=(True, False),
                encoder_temporal_down_sample=(True, False), encoder_block_dropout=(0.0, 0.0),
                decoder_layers_per_block=(1, 1), decoder_up_block_types=("UpDecoderBlockCausal3D",) * 2,
                decoder_block_out_channels=(64, 128), decoder_spatial_up_sample=(True, False),
                decoder_temporal_up_sample=(True, False), decoder_block_dropout=(0.0, 0.0), downsample_scale=2)


def _tiny_vae():
    return _reference_vae_cls()(**TINY_VAE)


def test_install_patches_every_causal_conv_and_uninstall_restores():
    vae = _tiny_vae()
    convs = VT.causal_convs(vae)
    names = {n for n, _ in convs}
    assert {"encoder.conv_in", "encoder.conv_out", "decoder.conv_in", "decoder.conv_out", "quant_conv", "post_quant_conv",
            "decoder.up_blocks.1.resnets.0.conv_shortcut"} <= names
    strides = {tuple(m.conv.stride) for _, m in convs}
    assert strides == {(1, 1, 1), (1, 2, 2), (2, 1, 1)}
    before = {n: m.forward for n, m in vae.named_modules()}
    VT.install_training_convs(vae)
    for n, m in vae.named_modules():
        if n in names:
            assert m.__dict__.get("forward") is not None and m.forward.__func__ is VT._patched_forward, n
        else:
            assert "forward" not in m.__dict__ and m.forward == before[n], n    # GroupNorm, attention, Conv3d stay torch
    VT.uninstall_training_convs(vae)
    for n, m in vae.named_modules():
        assert "forward" not in m.__dict__ and m.forward == before[n], n
        assert not hasattr(m, VT._MARK)


def test_install_through_the_loss_wrapper_patches_its_vae():
    vae = _tiny_vae()

    class Wrapper(torch.nn.Module):            # CausalVideoVAELossWrapper's shape: the model is `.vae`
        def __init__(self, v):
            super().__init__()
            self.vae = v

    wrapper = Wrapper(vae)
    VT.install_training_convs(wrapper)
    assert vae.encoder.conv_in.forward.__func__ is VT._patched_forward
    VT.uninstall_training_convs(wrapper)
    assert "forward" not in vae.encoder.conv_in.__dict__


@pytest.mark.parametrize("change, match", [
    (lambda m: setattr(m.conv, "kernel_size", (3, 1, 1)), "kernel"),
    (lambda m: setattr(m.conv, "stride", (2, 2, 2)), "stride"),
    (lambda m: setattr(m.conv, "dilation", (1, 2, 2)), "dilation"),
    (lambda m: setattr(m, "pad_mode", "replicate"), "pad_mode"),
])
def test_install_refusals(change, match):
    vae = _tiny_vae()
    change(vae.decoder.conv_in)
    with pytest.raises(ValueError, match=match):
        VT.install_training_convs(vae)
    assert all("forward" not in m.__dict__ for _, m in VT.causal_convs(vae))      # nothing half-installed


def test_install_refuses_context_parallel(monkeypatch):
    vae = _tiny_vae()
    mod = type(vae.encoder.conv_in).forward.__globals__
    monkeypatch.setitem(mod, "is_context_parallel_initialized", lambda: True)
    with pytest.raises(ValueError, match="context-parallel"):
        VT.install_training_convs(vae)


def test_install_refuses_a_model_without_causal_convs():
    with pytest.raises(ValueError, match="CausalConv3d"):
        VT.install_training_convs(torch.nn.Sequential(torch.nn.Conv3d(3, 3, 3)))


def test_temporal_chunk_and_cpu_tensors_raise():
    vae = _tiny_vae()
    VT.install_training_convs(vae)
    x = torch.randn(1, 3, 1, 8, 8)
    with pytest.raises(ValueError, match="temporal-chunk"):
        vae.encoder.conv_in(x, is_init_image=True, temporal_chunk=True)
    with pytest.raises(RuntimeError, match="CPU"):
        vae.encoder.conv_in(x)
    with pytest.raises(RuntimeError, match="CPU"):
        VT.causal_conv3d(x, vae.encoder.conv_in.conv.weight, None)


@pytest.mark.parametrize("hw", [(9, 8), (8, 9)])
def test_odd_spatial_size_under_spatial_stride_raises(hw):
    x = torch.randn(1, 4, 3, *hw)
    with pytest.raises(ValueError, match="even H and W"):
        VT.causal_conv3d(x, torch.randn(4, 4, 3, 3, 3), None, (1, 2, 2))
