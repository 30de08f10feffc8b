"""Per-kernel parity of the causal-VAE's HBM-bound kernels (pf_vae_elementwise.cu: GroupNorm statistics and apply, row
softmax, latent packing, tile blending) and of the conv store options the decode and encode rely on (fp32 / bf16 /
uint8 stores, partial channel stores, residual from a halo'd buffer).  Each kernel is called through the C ABI and
compared with a plain fp64 reference of the same operation; output buffers start out holding a sentinel so that what a
kernel must not write can be checked.  Needs an H100."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = 7.0
GN_EPS = 1e-6          # the decoder's GroupNorm eps (vae._gn)


def _lib():
    from pyramid_flow_b200 import _lib
    _lib.require_device()
    return _lib


def _ulp_bf16(ref: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |ref| (8 significant bits; 2^-133 below the normal range)."""
    _, e = torch.frexp(ref.abs().double())
    return torch.where(ref == 0, 2.0 ** -133, torch.ldexp(torch.ones_like(ref, dtype=torch.float64), e - 8)).clamp_min(2.0 ** -133)


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm
# ---------------------------------------------------------------------------------------------------------------------
GN_RATIOS = (0.0, 3.0, 30.0, 100.0)    # group |mean| / std, cycled over the groups; the last group is constant


def _gn_input(frames, voxels, c, groups, seed):
    """bf16 [frames, voxels, c]: per group a scale, a mean of GN_RATIOS[g % 4] group stds, and per-channel means spread
    inside the group (so the between-channel spread is part of the group variance); the last group is one constant."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    cpg = c // groups
    scale = torch.exp2(torch.randint(-4, 5, (groups,), generator=g, device=DEV).float())        # 1/16 .. 16
    ratio = torch.tensor([GN_RATIOS[i % len(GN_RATIOS)] for i in range(groups)], device=DEV)
    sign = torch.where(torch.rand(groups, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    spread = 0.7                                                                                   # channel means / noise std
    gmean = sign * ratio * scale * (1 + spread ** 2) ** 0.5
    cmean = gmean.repeat_interleave(cpg) + spread * scale.repeat_interleave(cpg) * torch.randn(c, generator=g, device=DEV)
    x = torch.randn(frames, voxels, c, generator=g, device=DEV) * scale.repeat_interleave(cpg) + cmean
    x[:, :, (groups - 1) * cpg:] = 2.5
    return x.bfloat16()


def _gn_ref(x, groups):
    """fp64 two-pass mean and population variance per (frame, group) of the bf16 input: [frames, groups] each."""
    frames, voxels, c = x.shape
    means, variances = [], []
    for f in range(frames):                    # one frame at a time: a 768x1280x128 frame is 1 GiB in fp64
        xf = x[f].view(voxels, groups, c // groups).double()
        m = xf.mean(dim=(0, 2))
        variances.append(((xf - m[None, :, None]) ** 2).mean(dim=(0, 2)))
        means.append(m)
        del xf
    return torch.stack(means), torch.stack(variances)


def _gn_ws_floats(frames, voxels, c):
    return frames * min(64, max(1, (voxels + 4095) // 4096)) * c * 2


def _gn_stats(x, groups, ws_floats=None, eps=GN_EPS):
    lib = _lib()
    frames, voxels, c = x.shape
    stats = torch.full((frames, groups, 2), SENTINEL, device=DEV)
    n = _gn_ws_floats(frames, voxels, c) if ws_floats is None else ws_floats
    ws = torch.empty(max(n, 1), device=DEV)
    lib.check(lib.load().pf_groupnorm_stats(x.data_ptr(), frames, voxels, c, groups, eps, stats.data_ptr(), ws.data_ptr(),
                                            n, lib.stream_ptr()), "pf_groupnorm_stats")
    torch.cuda.synchronize()
    return stats


@pytest.mark.parametrize("frames,voxels,c", [
    (3, 96, 512),             # nsplit = 1
    (2, 561, 128),            # ragged voxel count
    (2, 4097, 384),           # two splits with a ragged boundary; C/8 = 48 does not divide the 256-thread block
    (1, 1000, 2048),          # one voxel lane per block (vstep = 1)
    (2, 245760, 256),         # 384x640 frames
    (1, 983040, 128),         # 768x1280 frame: nsplit capped at 64
])
def test_groupnorm_stats_vs_fp64(frames, voxels, c):
    groups = 32
    x = _gn_input(frames, voxels, c, groups, seed=voxels + c)
    mean, var = _gn_ref(x, groups)
    stats = _gn_stats(x, groups).double()
    std, rstd = var.sqrt(), (var + torch.tensor(GN_EPS, dtype=torch.float32).double()).rsqrt()
    dmean = (stats[..., 0] - mean).abs()
    drstd = (stats[..., 1] - rstd).abs() / rstd
    ratio = torch.tensor([GN_RATIOS[i % len(GN_RATIOS)] for i in range(groups)], device=DEV)
    worst = {r: f"{drstd[:, ratio == r].max().item():.2e}" for r in GN_RATIOS}
    assert bool((dmean <= 1e-5 * std + 2.0 ** -23 * mean.abs()).all()), \
        f"mean error {(dmean / (std + 1e-30)).max().item():.2e} std; rstd error by |mean|/std: {worst}"
    assert bool((drstd <= 1e-5).all()), f"rstd relative error by |mean|/std: {worst}, constant group {drstd[:, -1].max().item():.2e}"
    assert torch.equal(stats[:, -1, 0], mean[:, -1]), "constant group: mean is the constant"


def test_groupnorm_stats_chunk_invariant():
    """Statistics of T frames from one call are bit-identical to T one-frame calls: the chunked decode depends on it."""
    x = _gn_input(3, 9000, 256, 32, seed=5)
    whole = _gn_stats(x, 32)
    for f in range(3):
        assert torch.equal(_gn_stats(x[f:f + 1], 32)[0], whole[f]), f


def test_groupnorm_stats_refuses_bad_arguments():
    lib = _lib()
    x = torch.zeros(2, 5000, 64, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="workspace"):
        _gn_stats(x, 32, ws_floats=_gn_ws_floats(2, 5000, 64) - 1)
    for c, groups in ((60, 30), (64, 24)):                  # C % 8 != 0, C % groups != 0
        y = torch.zeros(2, 100, c, device=DEV, dtype=torch.bfloat16)
        with pytest.raises(RuntimeError):
            _gn_stats(y, groups)
    assert lib.load().pf_groupnorm_stats(x.data_ptr(), 2, 5000, 64, 32, GN_EPS, None, None, 0, lib.stream_ptr()) != 0


def test_groupnorm_refuses_empty_shapes():
    """groups = 0 and voxels = 0 are refused before any division or any read of the first voxel."""
    x = torch.zeros(1, 16, 64, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        _gn_stats(x, 0)
    with pytest.raises(RuntimeError):
        _gn_stats(x[:, :0], 32, ws_floats=1024)
    lib = _lib()
    stats = torch.zeros(1, 32, 2, device=DEV)
    gb = torch.zeros(64, device=DEV)
    with pytest.raises(RuntimeError):
        lib.check(lib.load().pf_groupnorm_apply(x.data_ptr(), x.data_ptr(), 1, 1, 16, 64, 0, stats.data_ptr(), gb.data_ptr(),
                                                gb.data_ptr(), 0, 1, 0, lib.stream_ptr()), "pf_groupnorm_apply")


def _gn_apply(x, stats, gamma, beta, b, t, silu, groups=32):
    """x bf16 [b*t, voxels, c] -> y bf16 [b, t + 2, voxels, c], data in frames [2, t + 2), sentinel in the halo."""
    lib = _lib()
    _, voxels, c = x.shape
    y = torch.full((b, t + 2, voxels, c), SENTINEL, device=DEV, dtype=torch.bfloat16)
    lib.check(lib.load().pf_groupnorm_apply(x.data_ptr(), y.data_ptr(), b, t, voxels, c, groups, stats.data_ptr(),
                                            gamma.data_ptr(), beta.data_ptr(), int(silu), t + 2, 2, lib.stream_ptr()),
              "pf_groupnorm_apply")
    torch.cuda.synchronize()
    return y


def _gn_apply_ref(x, mean, rstd, gamma, beta, silu, groups=32):
    """fp64 GroupNorm(+SiLU) of x [F, V, C] with per-(frame, group) mean / rstd [F, G]; also returns the magnitude of the
    terms that are summed, |(x - mean) rstd gamma| + |beta|, for the fp32 rounding slack of outputs that cancel to ~0."""
    cpg = x.shape[-1] // groups
    m = mean.double().repeat_interleave(cpg, dim=1)[:, None]
    r = rstd.double().repeat_interleave(cpg, dim=1)[:, None]
    p = (x.double() - m) * r * gamma.double()
    v = p + beta.double()
    if silu:
        v = v * torch.sigmoid(v)
    return v, p.abs() + beta.double().abs()


@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_apply_vs_fp64(silu):
    """Apply judged alone: it gets the fp64 statistics rounded to fp32, and the reference uses those same fp32 values.
    Output = bf16(fp64 reference) on >= 99.9% of elements; elsewhere within 1 bf16 ulp, plus, for outputs that cancel
    to ~0 (|(x - mean) rstd gamma| ~ |beta|), a few fp32 ulps of the summed terms."""
    b, t, voxels, c, groups = 2, 3, 561, 256, 32
    x = _gn_input(b * t, voxels, c, groups, seed=11)
    g = torch.Generator(device=DEV).manual_seed(12)
    gamma = 1 + 0.5 * torch.randn(c, generator=g, device=DEV)
    beta = 0.5 * torch.randn(c, generator=g, device=DEV)
    mean, var = _gn_ref(x, groups)
    stats = torch.stack([mean, (var + GN_EPS).rsqrt()], -1).float().contiguous()
    y = _gn_apply(x, stats, gamma, beta, b, t, silu)
    assert bool((y[:, :2] == SENTINEL).all()), "halo frames must stay untouched"
    ref, mag = _gn_apply_ref(x, stats[..., 0], stats[..., 1], gamma, beta, silu)
    ref, mag = ref.view(b, t, voxels, c), mag.view(b, t, voxels, c)
    out = y[:, 2:].double()
    err = (out - ref).abs()
    bound = _ulp_bf16(ref) + 2.0 ** -20 * mag
    assert bool((err <= bound).all()), f"worst error {(err / _ulp_bf16(ref)).max().item():.2f} bf16 ulps"
    exact = (y[:, 2:] == ref.to(torch.bfloat16)).double().mean().item()
    assert exact >= 0.999, exact


def test_groupnorm_end_to_end_vs_fp64():
    """Stats + apply (SiLU) from the kernel's own statistics against an fp64 GroupNorm: within 1 bf16 ulp plus what the
    statistics' stated accuracy (mean 1e-5 std + 2^-23 |mean|, rstd 1e-5) moves the output."""
    b, t, voxels, c, groups = 1, 2, 24576, 128, 32
    x = _gn_input(b * t, voxels, c, groups, seed=21)
    g = torch.Generator(device=DEV).manual_seed(22)
    gamma = 1 + 0.5 * torch.randn(c, generator=g, device=DEV)
    beta = 0.5 * torch.randn(c, generator=g, device=DEV)
    y = _gn_apply(x, _gn_stats(x, groups), gamma, beta, b, t, True)
    mean, var = _gn_ref(x, groups)
    rstd = (var + GN_EPS).rsqrt()
    ref, mag = _gn_apply_ref(x, mean, rstd, gamma, beta, True)
    cpg = c // groups
    xn = ((x.double() - mean.repeat_interleave(cpg, 1)[:, None]) * rstd.repeat_interleave(cpg, 1)[:, None]).abs()
    shift = (1e-5 + 2.0 ** -23 * (mean.abs() * rstd).repeat_interleave(cpg, 1)[:, None] + 1e-5 * xn) * gamma.double().abs()
    err = (y[0, 2:].double() - ref).abs()
    bound = _ulp_bf16(ref) + 2.0 ** -20 * mag + 1.1 * shift
    assert bool((err <= bound).all()), f"worst error {(err / _ulp_bf16(ref)).max().item():.2f} bf16 ulps"


# ---------------------------------------------------------------------------------------------------------------------
# Row softmax (mid-block attention)
# ---------------------------------------------------------------------------------------------------------------------
def _softmax_case(rows, cols, ld, scale, scores):
    """Run pf_softmax_rows on `scores` [rows, cols] inside a sentinel-filled [rows + 1, ld] buffer; check the padding
    columns become 0, the row after `rows` stays untouched and |p - fp64 softmax| <= 1 bf16 ulp.  Returns p [rows, cols]."""
    lib = _lib()
    buf = torch.full((rows + 1, ld), SENTINEL, device=DEV, dtype=torch.bfloat16)
    buf[:rows, :cols] = scores
    lib.check(lib.load().pf_softmax_rows(buf.data_ptr(), rows, cols, ld, scale, lib.stream_ptr()), "pf_softmax_rows")
    torch.cuda.synchronize()
    assert bool((buf[:rows, cols:] == 0).all()), "padding columns must be zero"
    assert bool((buf[rows] == SENTINEL).all()), "the row after the last must stay untouched"
    p = buf[:rows, :cols]
    s32 = torch.tensor(scale, dtype=torch.float32).item()       # the kernel's fp32 scale
    for r0 in range(0, rows, 500):                               # fp64 reference a slab of rows at a time
        ref = torch.softmax(scores[r0:r0 + 500].double() * s32, dim=-1)
        err = (p[r0:r0 + 500].double() - ref).abs()
        assert bool((err <= _ulp_bf16(ref)).all()), f"rows {r0}+: worst error {(err / _ulp_bf16(ref)).max().item():.2f} bf16 ulps"
    return p


@pytest.mark.parametrize("rows,cols,ld", [(96, 96, 128), (561, 561, 576), (1000, 1000, 1024), (2000, 15360, 15360)])
def test_softmax_rows_vs_fp64(rows, cols, ld):
    """Mid-block attention shapes (scale 512^-0.5); the last is 2000 rows of the full-size 96x160-latent frame.  Row
    sharpness varies from flat to peaked: the score std per row runs from 1 to 100."""
    g = torch.Generator(device=DEV).manual_seed(rows)
    sd = torch.logspace(0, 2, rows, device=DEV)[:, None]
    scores = (torch.randn(rows, cols, generator=g, device=DEV) * sd).bfloat16()
    _softmax_case(rows, cols, ld, 512 ** -0.5, scores)


def test_softmax_rows_edges():
    # one column: every probability is exactly 1
    p = _softmax_case(37, 1, 64, 512 ** -0.5, torch.randn(37, 1, device=DEV).bfloat16())
    assert bool((p == 1).all())
    # a constant row: exactly uniform
    p = _softmax_case(5, 300, 320, 512 ** -0.5, torch.full((5, 300), 3.0, device=DEV).bfloat16())
    assert bool((p == p[0, 0]).all())
    # scale 1 and one score 100 above the rest: exactly one-hot
    s = (0.5 * torch.randn(8, 1000, device=DEV)).clamp(-4, 4).bfloat16()
    hot = torch.arange(8, device=DEV) * 123
    s[torch.arange(8, device=DEV), hot] = 104.0
    p = _softmax_case(8, 1000, 1024, 1.0, s)
    assert torch.equal(p.float(), F.one_hot(hot, 1000).float())


# ---------------------------------------------------------------------------------------------------------------------
# Latent packing
# ---------------------------------------------------------------------------------------------------------------------
def _pack(z, cpad, y_t_total, y_t_offset, fs=None, fh=None):
    lib = _lib()
    b, c, t, h, w = z.shape
    y = torch.full((b, y_t_total, h, w, cpad), SENTINEL, device=DEV, dtype=torch.bfloat16)
    lib.check(lib.load().pf_pack_latent(z.data_ptr(), int(z.dtype == torch.float32), b, c, t, h, w, y.data_ptr(), cpad,
                                        y_t_total, y_t_offset, None if fs is None else fs.data_ptr(),
                                        None if fh is None else fh.data_ptr(), lib.stream_ptr()), "pf_pack_latent")
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_pack_latent(dtype):
    b, c, t, h, w, cpad = 2, 16, 3, 11, 13, 64
    g = torch.Generator(device=DEV).manual_seed(3)
    z = (torch.randn(b, c, t, h, w, generator=g, device=DEV) * 2).to(dtype)
    zl = z.permute(0, 2, 3, 4, 1)                                   # [b, t, h, w, c]
    y = _pack(z, cpad, t + 2, 2)
    assert torch.equal(y[:, 2:, ..., :c], zl.to(torch.bfloat16)), "plain packing is a bit-exact bf16 rounding"
    assert bool((y[:, 2:, ..., c:] == 0).all()) and bool((y[:, :2] == SENTINEL).all())
    fs = 1 / (0.5 + torch.rand(t, generator=g, device=DEV))
    fh = torch.randn(t, generator=g, device=DEV)
    y = _pack(z, cpad, t + 2, 2, fs, fh)
    assert bool((y[:, 2:, ..., c:] == 0).all()) and bool((y[:, :2] == SENTINEL).all())
    ref = zl.double() * fs.double()[None, :, None, None, None] + fh.double()[None, :, None, None, None]
    out = y[:, 2:, ..., :c]
    err = (out.double() - ref).abs()
    assert bool((err <= _ulp_bf16(ref)).all()), f"worst error {(err / _ulp_bf16(ref)).max().item():.2f} bf16 ulps"
    assert (out == ref.to(torch.bfloat16)).double().mean().item() >= 0.999


def test_pack_latent_refuses_bad_arguments():
    z = torch.zeros(1, 16, 2, 4, 4, device=DEV)
    with pytest.raises(RuntimeError):
        _pack(z, 8, 2, 0)                      # cpad < c
    with pytest.raises(RuntimeError):
        _pack(z, 64, 3, 2)                     # frames [2, 4) outside a 3-frame buffer
    lib = _lib()
    y = torch.zeros(1, 4, 4, 4, 64, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        lib.check(lib.load().pf_pack_latent(z.data_ptr(), 1, 1, 16, 2, 4, 4, y.data_ptr(), 64, 4, -1, None, None,
                                            lib.stream_ptr()), "pf_pack_latent")


# ---------------------------------------------------------------------------------------------------------------------
# Tile blending (tiled decode / encode)
# ---------------------------------------------------------------------------------------------------------------------
def _blend_ref(a, b, extent, dim):
    """blend_v / blend_h of the reference VAE in fp64: b[.., y, ..] = a[.., la - extent + y, ..] (1 - y/extent)
    + b[.., y, ..] y/extent for y < extent."""
    out = b.double().clone()
    la = a.shape[dim]
    for y in range(extent):
        wgt = y / extent
        out.select(dim, y).copy_(a.double().select(dim, la - extent + y) * (1 - wgt) + b.double().select(dim, y) * wgt)
    return out


def _blend_raw(a, b, extent, dim):
    lib = _lib()
    outer = int(torch.tensor(b.shape[:dim]).prod().item())
    inner = int(torch.tensor(b.shape[dim + 1:]).prod().item())
    lib.check(lib.load().pf_blend_tiles(a.data_ptr(), b.data_ptr(), outer, a.shape[dim], b.shape[dim], inner, extent,
                                        lib.stream_ptr()), "pf_blend_tiles")
    torch.cuda.synchronize()


@pytest.mark.parametrize("dim", [3, 4])
@pytest.mark.parametrize("extent", [1, 8, 24])
def test_blend_tiles_vs_fp64(dim, extent):
    """5-D fp32 tiles [B, C, T, H, W] blended along H or W, la = 24 and lb = 40 > extent.  The blend is a convex
    combination, so the error is held to 2 fp32 ulps (2^-23 relative each) of |a| + |b|; the rows of b at or beyond
    `extent` and all of a stay bit-unchanged."""
    g = torch.Generator(device=DEV).manual_seed(extent * 10 + dim)
    shape_a, shape_b = [2, 3, 2, 20, 28], [2, 3, 2, 20, 28]
    shape_a[dim], shape_b[dim] = 24, 40
    a = torch.randn(*shape_a, generator=g, device=DEV)
    b = torch.randn(*shape_b, generator=g, device=DEV)
    a0, b0 = a.clone(), b.clone()
    ref = _blend_ref(a, b, extent, dim)
    _blend_raw(a, b, extent, dim)
    assert torch.equal(a, a0)
    assert torch.equal(b.narrow(dim, extent, 40 - extent), b0.narrow(dim, extent, 40 - extent))
    mag = (a.double().narrow(dim, 24 - extent, extent).abs() + b0.double().narrow(dim, 0, extent).abs())
    err = (b.narrow(dim, 0, extent).double() - ref.narrow(dim, 0, extent)).abs()
    assert bool((err <= 2 * 2.0 ** -23 * mag).all()), (err / mag).max().item()
    # vae._blend: the same kernel, extent clamped to both tiles
    from pyramid_flow_b200.vae import _blend
    b2 = b0.clone()
    assert _blend(a, b2, extent, dim) is b2 and torch.equal(b2, b)
    b3, b4 = b0.clone(), b0.clone()
    _blend(a, b3, 100, dim)
    _blend_raw(a, b4, 24, dim)
    assert torch.equal(b3, b4)


def test_blend_tiles_refuses_bad_extent():
    a = torch.zeros(1, 8, 4, device=DEV)
    b = torch.zeros(1, 16, 4, device=DEV)
    for extent in (9, 0):                      # extent > la, extent = 0
        with pytest.raises(RuntimeError):
            _blend_raw(a, b, extent, 1)
    with pytest.raises(RuntimeError):          # extent > lb
        _blend_raw(b, a, 12, 1)


# ---------------------------------------------------------------------------------------------------------------------
# Conv store options (pf_causal_conv3d): fp32 / bf16 / uint8 stores of one accumulator, partial channel stores, residual
# ---------------------------------------------------------------------------------------------------------------------
def _conv_setup(ci, co, k, t, h, w, seed):
    """A _Conv with bf16-exact weights, and its bf16 input [t + k - 1, h, w, cin_p] with a zero causal halo."""
    from pyramid_flow_b200.vae import _Conv
    g = torch.Generator().manual_seed(seed)
    wt = (torch.randn(co, ci, k, k, k, generator=g) * (ci * k ** 3) ** -0.5).bfloat16().float()
    bias = torch.randn(co, generator=g) * 0.1
    cv = _Conv({"c.conv.weight": wt, "c.conv.bias": bias}, "c", torch.device(DEV))
    xin = torch.zeros(t + k - 1, h, w, cv.cin_p, dtype=torch.bfloat16)
    xin[k - 1:, ..., :ci] = torch.randn(t, h, w, ci, generator=g).bfloat16()
    return cv, wt, bias, xin.to(DEV)


def _conv_ref64(xin, ci, wt, bias, k):
    """fp64 causal conv (on the CPU) of the halo'd channels-last input -> [t, h, w, co]."""
    x = xin[..., :ci].permute(3, 0, 1, 2)[None].double().cpu()
    x = F.pad(x, (k // 2, k // 2, k // 2, k // 2))
    return F.conv3d(x, wt.double(), bias.double())[0].permute(1, 2, 3, 0)


def _conv(cv, xin, t, h, w, out, **kw):
    from pyramid_flow_b200.vae import B200CausalVAE
    holder = B200CausalVAE.__new__(B200CausalVAE)          # only the _conv wrapper is needed
    B200CausalVAE._conv(holder, cv, xin, t, h, w, out=out, **kw)
    torch.cuda.synchronize()
    return out


def test_conv_out_store_modes():
    """decoder.conv_out (3x3x3, 128 -> 3, filters padded to 64): the fp32, bf16 and uint8 stores of one run are the same
    accumulators, so bf16 = bf16(fp32) and uint8 = trunc(clamp(fmaf(fp32, 127.5, 127.5), 0, 255)) bit for bit."""
    t, h, w = 2, 12, 40
    cv, wt, bias, xin = _conv_setup(128, 3, 3, t, h, w, seed=1)
    f32 = _conv(cv, xin, t, h, w, torch.full((t, h, w, 3), SENTINEL, device=DEV), store_channels=3, out_f32=1)
    bf = _conv(cv, xin, t, h, w, torch.full((t, h, w, 3), SENTINEL, device=DEV, dtype=torch.bfloat16), store_channels=3)
    u8 = _conv(cv, xin, t, h, w, torch.full((t, h, w, 3), 7, device=DEV, dtype=torch.uint8), store_channels=3, out_f32=2)
    ref = _conv_ref64(xin, 128, wt, bias, 3)
    assert (f32.double().cpu() - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()
    assert torch.equal(bf, f32.to(torch.bfloat16))
    # v * 127.5 + 127.5 is exact in fp64 unless |v| is tiny (the product has 24 + 8 significant bits); rounding it to fp32
    # is what fmaf returns, and the kernel truncates that
    img = (f32.double() * 127.5 + 127.5).float().clamp(0, 255).floor().to(torch.uint8)
    assert torch.equal(u8, img)
    assert bool((u8 == 0).any()) and bool((u8 == 255).any()), "the data must reach both clamps"
    # out_c = 8, store_channels = 3: channels 3..7 keep the sentinel
    wide = _conv(cv, xin, t, h, w, torch.full((t, h, w, 8), SENTINEL, device=DEV, dtype=torch.bfloat16), store_channels=3)
    assert torch.equal(wide[..., :3], bf) and bool((wide[..., 3:] == SENTINEL).all())


def test_conv_quant_conv_fp32_partial_store():
    """quant_conv: 1x1x1, fp32 store of 32 of the 64 padded filters into a 32-channel buffer."""
    t, h, w = 3, 9, 21
    cv, wt, bias, xin = _conv_setup(32, 32, 1, t, h, w, seed=2)
    out = _conv(cv, xin, t, h, w, torch.full((t, h, w, 32), SENTINEL, device=DEV), store_channels=32, out_f32=1)
    ref = _conv_ref64(xin, 32, wt, bias, 1)
    assert (out.double().cpu() - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()


def test_conv_residual_from_halo_buffer():
    """Residual read from frames [2, t + 2) of a halo'd buffer (res_t_total = t + 2, res_t_offset = 2) whose halo
    frames hold large values: bf16(acc + res) and acc + res in fp32, bit for bit against the plain fp32 store."""
    t, h, w = 2, 10, 33
    cv, wt, bias, xin = _conv_setup(128, 128, 3, t, h, w, seed=3)
    acc = _conv(cv, xin, t, h, w, torch.zeros(t, h, w, 128, device=DEV), out_f32=1)
    res = torch.randn(t + 2, h, w, 128, device=DEV).bfloat16()
    res[:2] = 1000.0
    out = _conv(cv, xin, t, h, w, torch.zeros(t, h, w, 128, device=DEV, dtype=torch.bfloat16), residual=res, res_t_offset=2)
    assert torch.equal(out, (acc + res[2:].float()).to(torch.bfloat16))
    out32 = _conv(cv, xin, t, h, w, torch.zeros(t, h, w, 128, device=DEV), out_f32=1, residual=res, res_t_offset=2)
    assert torch.equal(out32, acc + res[2:].float())


def test_conv_refuses_bad_store_options():
    t, h, w = 1, 4, 8
    cv, _, _, xin = _conv_setup(64, 256, 3, t, h, w, seed=4)
    with pytest.raises(RuntimeError):          # spatial depth-to-space store is bf16 only
        _conv(cv, xin, t, h, w, torch.zeros(t, 2 * h, 2 * w, 64, device=DEV), store_mode=1, out_f32=1)
    res = torch.zeros(t, h, w, 256, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):          # the uint8 image store takes no residual
        _conv(cv, xin, t, h, w, torch.zeros(t, h, w, 256, device=DEV, dtype=torch.uint8), out_f32=2, residual=res)
