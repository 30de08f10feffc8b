"""Every conv kernel the VAE number rests on, pinned one by one through pf_conv3d_desc.kernel_variant (1 = 128-wide filter
tiles, 2 = 64-wide filter tiles) at shapes with >= 3 tiles along W (halo reuse across W tiles),
ragged last tiles, and at the headline layer shapes (128->128 @768x1280, 256->256 @384x640: sampled voxels vs fp32);
plus the full-resolution (96x160 latent) VAE decode against the fp32 oracle on the same GPU.  Needs an H100."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _mk(ci, co, dev, seed):
    from pyramid_flow_b200.vae import _Conv
    g = torch.Generator().manual_seed(seed)
    wt = (torch.randn(co, ci, 3, 3, 3, generator=g) * (ci * 27) ** -0.5).bfloat16().float()
    bias = torch.randn(co, generator=g) * 0.1
    return _Conv({"c.conv.weight": wt, "c.conv.bias": bias}, "c", dev), wt.to(dev), bias.to(dev)


def _run(cv, xin, t, h, w, co, variant, **kw):
    from pyramid_flow_b200.vae import B200CausalVAE
    holder = B200CausalVAE.__new__(B200CausalVAE)
    out = torch.zeros(t, h, w, co, device=xin.device, dtype=torch.bfloat16)
    B200CausalVAE._conv(holder, cv, xin, t, h, w, out=out, kernel_variant=variant, **kw)
    torch.cuda.synchronize()
    return out


def _sampled_err(x, wt, bias, out, n=8192):
    """max |out - conv(x)| over n output voxels incl. every border (x [T,H,W,Cin], causal 3x3x3, zero spatial pad), fp32."""
    t, h, w, ci = x.shape
    dev = x.device
    g = torch.Generator(device=dev).manual_seed(0)
    ts = torch.randint(0, t, (n,), device=dev, generator=g)
    hs = torch.randint(0, h, (n,), device=dev, generator=g)
    ws = torch.randint(0, w, (n,), device=dev, generator=g)
    k = n // 8
    hs[:k] = torch.where(torch.arange(k, device=dev) % 2 == 0, 0, h - 1)
    ws[k:2 * k] = torch.where(torch.arange(k, device=dev) % 2 == 0, 0, w - 1)
    ws[2 * k:3 * k] = (torch.randint(1, max(2, w // 128 + 1), (k,), device=dev, generator=g) * 128 - torch.randint(0, 2, (k,), device=dev, generator=g)).clamp(0, w - 1)  # W-tile seams
    xp = F.pad(x.float(), (0, 0, 1, 1, 1, 1, 2, 0))
    acc = bias.float()[None].repeat(n, 1)
    for dt in range(3):
        for dh in range(3):
            for dw in range(3):
                acc += xp[ts + dt, hs + dh, ws + dw] @ wt[:, :, dt, dh, dw].float().t()
    return (out[ts, hs, ws].float() - acc).abs().max().item()


@pytest.mark.parametrize("ci,co,t,h,w", [(64, 128, 2, 5, 300), (128, 256, 3, 4, 417), (128, 128, 2, 12, 1280), (256, 512, 1, 7, 384)])
def test_conv_kernel_variants_multi_tile_w(ci, co, t, h, w):
    """>= 3 (up to 10) 128-voxel tiles along W, ragged last tile: every kernel vs F.conv3d, and both kernels give the
    SAME BITS (one K accumulation order), so the dispatch never changes results."""
    dev = torch.device("cuda:0")
    cv, wt, bias = _mk(ci, co, dev, seed=ci + w)
    torch.manual_seed(w)
    x = torch.randn(t, h, w, ci, device=dev).bfloat16()
    xin = torch.zeros(t + 2, h, w, ci, device=dev, dtype=torch.bfloat16)
    xin[2:] = x
    xr = F.pad(x.permute(3, 0, 1, 2)[None].float(), (1, 1, 1, 1, 2, 0))
    ref = F.conv3d(xr, wt, bias)[0].permute(1, 2, 3, 0)
    outs = {}
    for variant in (1, 2):
        outs[variant] = _run(cv, xin, t, h, w, co, variant)
        err = (outs[variant].float() - ref).abs().max().item()
        assert err < 3e-2, (variant, ci, co, w, err)
    assert torch.equal(outs[1], outs[2]), "kernel variants must agree bit for bit"
    auto = _run(cv, xin, t, h, w, co, 0)
    assert torch.equal(auto, outs[1])
    # residual + store into a haloed buffer
    res = torch.randn(t, h, w, co, device=dev).bfloat16()
    from pyramid_flow_b200.vae import B200CausalVAE
    holder = B200CausalVAE.__new__(B200CausalVAE)
    out2 = torch.zeros(t + 2, h, w, co, device=dev, dtype=torch.bfloat16)
    B200CausalVAE._conv(holder, cv, xin, t, h, w, out=out2, out_t_offset=2, residual=res, kernel_variant=2)
    torch.cuda.synchronize()
    assert (out2[2:].float() - (ref + res.float())).abs().max().item() < 4e-2 and bool((out2[:2] == 0).all())


@pytest.mark.parametrize("ci,co,t,h,w", [(128, 128, 2, 768, 1280), (256, 256, 2, 384, 640)])
def test_conv_headline_layer_shapes(ci, co, t, h, w):
    """The layers the decode time is made of (up3 128->128 at 768x1280, up2 256->256 at 384x640): the default dispatch
    and the 64-wide-tile kernel, verified on 8192 sampled voxels (borders and W-tile seams included) in fp32."""
    dev = torch.device("cuda:0")
    cv, wt, bias = _mk(ci, co, dev, seed=7)
    torch.manual_seed(3)
    x = torch.randn(t, h, w, ci, device=dev).bfloat16()
    xin = torch.zeros(t + 2, h, w, ci, device=dev, dtype=torch.bfloat16)
    xin[2:] = x
    o_auto = _run(cv, xin, t, h, w, co, 0)
    e = _sampled_err(x, wt, bias, o_auto)
    assert e < 3e-2, e
    o2 = _run(cv, xin, t, h, w, co, 2)
    assert torch.equal(o2, o_auto)
    assert bool(torch.isfinite(o_auto.float()).all())


def test_vae_decode_full_resolution_matches_oracle():
    """BASELINE configs[2] latent size: 96x160 latent, 3 latent frames -> 17 frames of 768x1280, default-width decoder, chunked
    decode (window 1) through the C-ABI vs the fp32 oracle (cuDNN fp32, TF32 off) on the same GPU."""
    from oracle import vae_oracle as VO
    from pyramid_flow_b200.vae import B200CausalVAE, VaeConfigB200
    dev = torch.device("cuda:0")
    cfg = VO.VaeDecoderConfig()
    params = VO.synthetic_vae_params(cfg, seed=31)
    g = torch.Generator().manual_seed(32)
    z = torch.randn(1, 16, 3, 96, 160, generator=g).bfloat16().float()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    vae = B200CausalVAE(VaeConfigB200(), params, device=dev)
    out = vae.decode(z.to(dev), temporal_chunk=True, window_size=1).sample.float().cpu()
    torch.cuda.synchronize()
    del vae
    torch.cuda.empty_cache()
    pd = {k: v.to(dev) for k, v in params.items()}
    with torch.no_grad():
        ref = VO.decode(pd, cfg, z.to(dev)).float().cpu()
        torch.cuda.empty_cache()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ref_bf16 = VO.decode(pd, cfg, z.to(dev).bfloat16()).float().cpu()
    err, mse = (out - ref).abs().max().item(), ((out - ref) ** 2).mean().item()
    e2, m2 = (ref_bf16 - ref).abs().max().item(), ((ref_bf16 - ref) ** 2).mean().item()
    print(f"VAE 96x160 latent -> {tuple(out.shape)}: ours vs fp32 oracle max_abs {err:.3e} mse {mse:.3e} | reference bf16 policy "
          f"max_abs {e2:.3e} mse {m2:.3e} | |ref| mean {ref.abs().mean():.3f}")
    assert out.shape == ref.shape == (1, 3, 17, 768, 1280)
    assert err < 8.8e-2 and mse < 7.3e-5
    assert mse <= 2.0 * m2 + 1e-5, "must be comparable to the reference's own bf16 error"
