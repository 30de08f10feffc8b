"""fp64 references, per-element error bounds and exact GEMM probe operands for the DiT and text-encoder row kernels
(pf_elementwise.cu: LN + AdaLN modulate, small-M linear, timestep sinusoid, patchify / unpatchify, CFG + Euler;
pf_text.cu: T5 RMSNorm rows, token embedding), with the tests that show each check is sharp, and the host-side argument
checks of those entries.  No GPU: tests/test_row_kernels_gpu.py imports the helpers and runs the kernels against them.

Every bf16 output is checked per element against
    |out - ref64| <= 1/2 ulp_bf16(|ref64| + e32) + e32,
where ref64 is the operation in fp64 and e32 bounds what the kernel's fp32 arithmetic may add before the one rounding
to bf16; e32 is derived per op in the docstring of its reference.  u = 2^-24 is the fp32 unit roundoff, and
gamma(k) = k u / (1 - k u) bounds a chain of k fp32 roundings.  Accuracies of CUDA library functions are the maximum
ulp errors the CUDA C++ Programming Guide lists (expf, sinf, cosf, erff, rsqrtf: 2 ulp each); the approximate MUFU
ex2 / rcp instructions are given 2^-21 relative each, a margin over their documented accuracy.  Index and byte kernels
must match bit for bit."""
import ctypes as C
import math

import pytest
import torch

from pyramid_flow_b200 import _lib

U = 2.0 ** -24               # fp32 unit roundoff
MUFU_REL = 2.0 ** -21        # ex2.approx / rcp.approx relative error budget
LIB_ULP = 2                  # expf, sinf, cosf, erff, rsqrtf: documented maximum ulp error


def gamma(k: int) -> float:
    return k * U / (1 - k * U)


def ulp_bf16(a: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |a|: 2^(floor(log2 |a|) - 7), and 2^-133 below the normal range."""
    _, e = torch.frexp(a.abs().double())
    return torch.ldexp(torch.ones_like(a, dtype=torch.float64), e - 8).clamp_min(2.0 ** -133)


def ulp_f32(a: torch.Tensor) -> torch.Tensor:
    _, e = torch.frexp(a.abs().double())
    return torch.ldexp(torch.ones_like(a, dtype=torch.float64), e - 24).clamp_min(2.0 ** -149)


def bf16_bound(ref: torch.Tensor, e32) -> torch.Tensor:
    """1/2 ulp_bf16(|ref| + e32) + e32: one rounding to bf16 after an fp32 result within e32 of ref."""
    e32 = torch.as_tensor(e32, dtype=torch.float64, device=ref.device).expand_as(ref)
    return 0.5 * ulp_bf16(ref.abs() + e32) + e32


def check_bound(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str) -> None:
    """Per element |out - ref| <= bound (NaN fails); the message names the count and the worst index."""
    diff = (out.double() - ref.double()).abs()
    excess = torch.nan_to_num(diff - bound, nan=math.inf)
    if bool((excess > 0).any()):
        flat = int(torch.argmax(excess))
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), excess.shape))
        raise AssertionError(f"{what}: {int((excess > 0).sum())} of {excess.numel()} elements outside the bound; worst at "
                             f"{idx}: out {out[idx].item()!r} ref {ref[idx].item()!r} bound {bound[idx].item():.3g}")


def check_bf16(out: torch.Tensor, ref: torch.Tensor, e32, what: str) -> None:
    check_bound(out, ref, bf16_bound(ref.double(), e32), what)


def check_equal(out: torch.Tensor, ref: torch.Tensor, what: str) -> None:
    """Bit equality (same dtype); the message names the first differing index."""
    assert out.dtype == ref.dtype and out.shape == ref.shape, (what, out.dtype, ref.dtype, out.shape, ref.shape)
    ob, rb = out.contiguous(), ref.contiguous()
    ib = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[ob.element_size()]
    neq = ob.view(ib) != rb.view(ib)
    if bool(neq.any()):
        idx = tuple(int(i) for i in torch.nonzero(neq)[0])
        raise AssertionError(f"{what}: {int(neq.sum())} of {neq.numel()} elements differ; first at {idx}: out {out[idx].item()!r} "
                             f"ref {ref[idx].item()!r}")


# ---------------------------------------------------------------------------------------------------------------------
# LN + AdaLN modulate (N:174, N:234, N:120, B:1022-1023, B:1035-1036), CLIP LayerNorm as shift = bias, scale = weight - 1
# ---------------------------------------------------------------------------------------------------------------------
def ln_modulate_ref(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, eps: float):
    """y = (x - mean) / sqrt(var + eps) * (1 + scale) + shift over the last dim, in fp64 -> (ref, e32).

    The kernel (one warp per row) forms mean32 = fl(sum)/n, d_i = fl(x_i - mean32), ss = sum d_i^2, rstd = rsqrtf(ss/n + eps)
    and y_i = ((d_i rstd) (1 + scale_i)) + shift_i, all in fp32.  With k = n/128 + 8 the longest chain of a row sum (n/128
    float4 per lane, two in-vector adds, five shuffle levels, the division):
      |mean32 - mean| <= dm = gamma(k) mean|x|;
      d_i = (x_i - mean) + (mean - mean32) + rho_i, |rho_i| <= u |d_i|: the shared offset cancels from sum (x_i - mean) d_i,
      so ss = n var (1 + theta) + n dm^2 with |theta| <= gamma(k + 1) + 2u;
      rstd32 = rstd (1 + eta), eta <= (gamma(k + 1) + 4u + dm^2 / (var + eps)) / 2 + 2 LIB_ULP u (/n, + eps, rsqrtf);
      y32 - y <= |1 + scale| rstd (|d_i| (eta + 3u) + dm (1 + u)) + u |y|  (two products, 1 + scale, the add).
    The dm term is what a large |mean| / std costs: fp32 cannot hold the mean closer than that."""
    x = x.double()
    n = x.shape[-1]
    mean = x.mean(-1, keepdim=True)
    d = x - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    g = 1.0 + scale.double()
    ref = d * rstd * g + shift.double()
    k = n // 128 + 8
    dm = gamma(k) * x.abs().mean(-1, keepdim=True)
    eta = 0.5 * (gamma(k + 1) + 4 * U + dm * dm / (var + eps)) + 2 * LIB_ULP * U
    e32 = 1.01 * (g.abs() * rstd * (d.abs() * (eta + 3 * U) + dm * (1 + U)) + U * ref.abs())
    return ref, e32


LN_RATIOS = (0.0, 1.0, 10.0, 100.0, 1000.0)       # row |mean| / std, cycled over the rows


def ln_rows(rows: int, dim: int, seed: int, device="cpu") -> torch.Tensor:
    """fp32 [rows, dim]: row r has |mean| / std = LN_RATIOS[r % 5] with a random sign and a scale 2^j (j in [-6, 6]); every
    seventh row carries three 1e4-std outliers."""
    g = torch.Generator(device=device).manual_seed(seed)
    std = torch.exp2(torch.randint(-6, 7, (rows, 1), generator=g, device=device).float())
    ratio = torch.tensor([LN_RATIOS[r % len(LN_RATIOS)] for r in range(rows)], device=device)[:, None]
    sign = torch.where(torch.rand(rows, 1, generator=g, device=device) < 0.5, -1.0, 1.0)
    x = torch.randn(rows, dim, generator=g, device=device) * std + sign * ratio * std
    for r in range(3, rows, 7):
        cols = torch.randint(0, dim, (3,), generator=g, device=device)
        x[r, cols] += 1e4 * std[r, 0] * torch.tensor([1.0, -1.0, 1.0], device=device)
    return x


def _ln_fp32(x, shift, scale, eps, single_pass=False):
    """The LN + modulate in fp32, two-pass as the kernel, or the single-pass E[x^2] - mean^2 variance."""
    n = x.shape[-1]
    mean = x.sum(-1, keepdim=True) / n
    if single_pass:
        var = (x * x).sum(-1, keepdim=True) / n - mean * mean
    else:
        var = ((x - mean) ** 2).sum(-1, keepdim=True) / n
    return ((x - mean) * torch.rsqrt(var.clamp_min(0) + eps) * (1 + scale) + shift).bfloat16()


def _ln_case(seed=0, rows=40, dim=1536):
    g = torch.Generator().manual_seed(seed)
    x = ln_rows(rows, dim, seed)
    shift = torch.randn(1, dim, generator=g) * 0.5
    scale = torch.randn(1, dim, generator=g) * 0.3
    return x, shift, scale


def _one_ulp_past(ref, bound, idx):
    """The bf16 value one bf16 ulp beyond ref + bound at idx."""
    t = ref[idx] + bound[idx]
    return (t + ulp_bf16(t)).to(torch.bfloat16)


def test_ln_checker_accepts_the_reference_and_an_fp32_two_pass():
    x, shift, scale = _ln_case()
    ref, e32 = ln_modulate_ref(x, shift, scale, 1e-6)
    check_bf16(ref.bfloat16(), ref, e32, "fp64 reference")
    check_bf16(_ln_fp32(x, shift, scale, 1e-6), ref, e32, "fp32 two-pass")


def test_ln_checker_is_sharp():
    x, shift, scale = _ln_case()
    ref, e32 = ln_modulate_ref(x, shift, scale, 1e-6)
    bound = bf16_bound(ref, e32)
    base = ref.bfloat16()
    for idx in ((0, 0), (4, 777), (39, 1535)):      # a row of each of a zero, a 1e3 and a 1e3 mean / std ratio
        out = base.clone()
        out[idx] = _one_ulp_past(ref, bound, idx)
        with pytest.raises(AssertionError, match=rf"worst at \({idx[0]}, {idx[1]}\)"):
            check_bf16(out, ref, e32, "one element one ulp past")
    with pytest.raises(AssertionError):
        check_bf16(torch.roll(base, 1, dims=0), ref, e32, "rows shifted by one")
    with pytest.raises(AssertionError):
        check_bf16(torch.roll(base, 1, dims=1), ref, e32, "columns shifted by one")
    with pytest.raises(AssertionError):     # without the 1 + of the modulate
        check_bf16(((x - x.mean(-1, keepdim=True)) * torch.rsqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-6) * scale
                    + shift).bfloat16(), ref, e32, "scale instead of 1 + scale")
    big = slice(4, 40, 5)                    # the |mean| / std = 1e3 rows
    with pytest.raises(AssertionError):
        check_bf16(_ln_fp32(x, shift, scale, 1e-6, single_pass=True)[big], ref[big], e32[big], "single-pass variance")


# ---------------------------------------------------------------------------------------------------------------------
# small-M linear (N:147,164,209,223,99,110; E:84-158, E:185-201)
# ---------------------------------------------------------------------------------------------------------------------
def silu64(x: torch.Tensor) -> torch.Tensor:
    x = x.double()
    return x * torch.sigmoid(x)


def silu_rel_err(x: torch.Tensor) -> torch.Tensor:
    """Relative error of the kernels' silu_f(x) = x rcp(1 + ex2(-log2e x)): the fp32 argument costs u |x| in 2^arg; ex2, rcp
    MUFU_REL each; 1 + ex2 and the final product u each."""
    return 2 * MUFU_REL + U * x.double().abs() + 2 * U


def small_linear_ref(x, w, bias, y0=None, *, act_in=0, act_out=0, round_in_bf16=False):
    """y = act_out(act_in(x) W^T + bias) (+ y0) in fp64 -> (ref, bound), fp32 outputs.

    The dot product runs in fp32 in some order: |err| <= gamma(k + 1) (sum |w| |x| + |bias|) (every partial sum rounded once
    per add, the bias add included).  act_in: silu_f is within silu_rel_err of silu; with round_in_bf16 the activated
    input is rounded to bf16, which, when silu_f and silu straddle a rounding boundary, may land one bf16 ulp from the
    rounding of the exact silu: each input carries ulp_bf16(silu) then.  Without act_in, the bf16 rounding of an fp32
    input is exact and the reference applies it too.  act_out: |silu'| <= 1.1 carries the sum's error, plus
    silu_rel_err of the output; accumulate adds y0 with one rounding.  The result is fp32: one more u |y|."""
    x64 = x.double()
    w64 = w.double()
    k = x.shape[-1]
    if act_in:
        xin = silu64(x64)
        xerr = silu_rel_err(x64) * xin.abs()
        if round_in_bf16:
            xin = xin.float().bfloat16().double()
            xerr = ulp_bf16(xin)
    else:
        xin = x64.float().bfloat16().double() if round_in_bf16 else x64
        xerr = torch.zeros_like(xin)
    b64 = torch.zeros(w.shape[0], dtype=torch.float64, device=x.device) if bias is None else bias.double()
    s = xin @ w64.t() + b64
    mag = xin.abs() @ w64.abs().t() + b64.abs()
    err = gamma(k + 1) * mag + xerr @ w64.abs().t()
    if act_out:
        v = silu64(s)
        err = 1.1 * err + silu_rel_err(s) * v.abs()
        s = v
    if y0 is not None:
        s = s + y0.double()
        err = err + U * s.abs()
    return s, 1.01 * (err + U * s.abs())


def _sl_case(m=3, k=264, n=40, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(m, k, generator=g) * 2, (torch.randn(n, k, generator=g) * 0.05).bfloat16(), torch.randn(n, generator=g),
            torch.randn(m, n, generator=g))


@pytest.mark.parametrize("act_in,act_out,acc,rnd", [(0, 0, 0, 0), (1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0), (0, 0, 0, 1),
                                                    (1, 1, 1, 1)])
def test_small_linear_checker_accepts_fp32_and_is_sharp(act_in, act_out, acc, rnd):
    x, w, b, y0 = _sl_case()
    ref, bound = small_linear_ref(x, w, b, y0 if acc else None, act_in=act_in, act_out=act_out, round_in_bf16=bool(rnd))
    check_bound(ref.float(), ref, bound, "fp64 reference")
    xi = x * torch.sigmoid(x) if act_in else x                    # the same op in fp32, torch's order
    if rnd:
        xi = xi.bfloat16().float()
    y = xi @ w.float().t() + b
    if act_out:
        y = y * torch.sigmoid(y)
    if acc:
        y = y0 + y
    check_bound(y, ref, bound, "fp32")
    out = ref.float()
    out[2, 17] = (ref[2, 17] + bound[2, 17] + ulp_f32(ref[2, 17] + bound[2, 17])).float()
    with pytest.raises(AssertionError, match=r"worst at \(2, 17\)"):
        check_bound(out, ref, bound, "one element one ulp past")
    with pytest.raises(AssertionError):
        check_bound(torch.roll(ref.float(), 1, dims=1), ref, bound, "columns shifted by one")
    with pytest.raises(AssertionError):
        check_bound(torch.roll(ref.float(), 1, dims=0), ref, bound, "rows shifted by one")


# ---------------------------------------------------------------------------------------------------------------------
# timestep sinusoid (E:11-62, flip_sin_to_cos=True, downscale_freq_shift=0)
# ---------------------------------------------------------------------------------------------------------------------
def timestep_ref(t: torch.Tensor, dim: int, round_bf16: bool):
    """-> (ref, bound) fp32 [m, dim] = [cos(t f_i), sin(t f_i)], f_i = exp(-ln(1e4) i / half).

    The exponent is formed in fp32 as the reference (and the kernel) forms it, (-ln(1e4) i) / half; from there everything
    is fp64.  The kernel's expf is within LIB_ULP fp32 ulps of exp, t f within one more rounding, so its argument is within
    |arg| (LIB_ULP 2u + u) of the exact t f_i; sin and cos move by at most that, and sinf / cosf add LIB_ULP ulps of the
    output.  With round_bf16 the output is then rounded to bf16."""
    half = dim // 2
    i = torch.arange(half, dtype=torch.float32, device=t.device)
    # tensor / tensor: an IEEE fp32 division (torch may multiply by the reciprocal of a Python scalar divisor)
    expo = (-math.log(10000.0) * i) / torch.full_like(i, half)
    arg = t.double()[:, None] * torch.exp(expo.double())[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], dim=-1)
    e = torch.cat([arg.abs(), arg.abs()], dim=-1) * (2 * LIB_ULP * U + U) * 1.01 + LIB_ULP * ulp_f32(ref)
    return ref, (bf16_bound(ref, e) if round_bf16 else e)


TIMESTEPS = (0.0, 0.5, 1.0, 999.0, 1000.0)


def test_timestep_checker_is_sharp():
    t = torch.tensor(TIMESTEPS + (972.0, 3.5, 0.25))
    for rnd in (False, True):
        ref, bound = timestep_ref(t, 256, rnd)
        base = ref.float().bfloat16().float() if rnd else ref.float()
        check_bound(base, ref, bound, "fp64 reference")
        arg32 = t[:, None] * torch.exp((-math.log(10000.0) * torch.arange(128, dtype=torch.float32)) / 128)[None]
        emb = torch.cat([arg32.cos(), arg32.sin()], -1)           # torch's fp32 formula
        check_bound(emb.bfloat16().float() if rnd else emb, ref, bound, "fp32")
        out = base.clone()
        out[4, 3] = (ref[4, 3] + bound[4, 3] + (ulp_bf16 if rnd else ulp_f32)(ref[4, 3] + bound[4, 3])).float()
        with pytest.raises(AssertionError, match=r"worst at \(4, 3\)"):
            check_bound(out, ref, bound, "one element one ulp past")
        with pytest.raises(AssertionError):     # sin first
            check_bound(torch.roll(base, 128, dims=1), ref, bound, "halves swapped")
        with pytest.raises(AssertionError):     # frequency index off by one
            check_bound(torch.cat([torch.roll(base[:, :128], 1, 1), base[:, 128:]], 1), ref, bound, "frequencies shifted")


# ---------------------------------------------------------------------------------------------------------------------
# CFG + Euler (P:771-776, S:278-286)
# ---------------------------------------------------------------------------------------------------------------------
def cfg_euler_ref(v2: torch.Tensor, guidance: float, dsigma: float, x: torch.Tensor):
    """x + dsigma (vu + g (vc - vu)) in fp64 -> (ref, bound): the fp32 kernel rounds vc - vu, the product by g, the add to
    vu, the product by dsigma and the final add (fused or not): each at most u of its result."""
    vu, vc = v2[0].double(), v2[1].double()
    diff = vc - vu
    v = vu + guidance * diff
    ref = x.double() + dsigma * v
    err_v = U * (2 * abs(guidance) * diff.abs() + v.abs())
    return ref, 1.01 * (abs(dsigma) * (err_v + U * v.abs()) + U * ref.abs())


def test_cfg_euler_checker_is_sharp():
    g = torch.Generator().manual_seed(3)
    v2, x = torch.randn(2, 1000, generator=g), torch.randn(1000, generator=g)
    ref, bound = cfg_euler_ref(v2, 5.0, -0.05, x)
    check_bound(x + (-0.05) * (v2[0] + 5.0 * (v2[1] - v2[0])), ref, bound, "fp32")
    out = ref.float()
    out[611] = (ref[611] + bound[611] + ulp_f32(ref[611] + bound[611])).float()
    with pytest.raises(AssertionError, match=r"worst at \(611,\)"):
        check_bound(out, ref, bound, "one element one ulp past")
    with pytest.raises(AssertionError):
        check_bound(x + (-0.05) * (v2[1] + 5.0 * (v2[0] - v2[1])), ref, bound, "uncond and cond swapped")


# ---------------------------------------------------------------------------------------------------------------------
# T5LayerNorm rows (T5 T5LayerNorm.forward)
# ---------------------------------------------------------------------------------------------------------------------
def rms_norm_ref(x: torch.Tensor, w: torch.Tensor, eps: float):
    """y = w x / sqrt(mean(x^2) + eps) in fp64 -> (ref, e32).  The kernel sums squares with a chain of k = n/128 + 9 (n/128
    float4 per lane, the product and two in-vector adds, five shuffle levels), then /n, + eps, rsqrtf (LIB_ULP ulps), and
    two products: rstd32 within (gamma(k) + 2u) / 2 + 2 LIB_ULP u, y within two more u."""
    x64 = x.double()
    n = x.shape[-1]
    ms = (x64 * x64).mean(-1, keepdim=True)
    ref = w.double() * x64 / torch.sqrt(ms + eps)
    k = n // 128 + 9
    eta = 0.5 * (gamma(k) + 2 * U) + 2 * LIB_ULP * U
    return ref, 1.01 * ref.abs() * (eta + 2 * U)


def test_rms_norm_checker_is_sharp():
    g = torch.Generator().manual_seed(4)
    x = torch.randn(12, 4100, generator=g) * torch.exp2(torch.randint(-8, 9, (12, 1), generator=g).float())
    w = 1 + 0.2 * torch.randn(4100, generator=g)
    ref, e32 = rms_norm_ref(x, w, 1e-6)
    check_bf16(ref.bfloat16(), ref, e32, "fp64 reference")
    check_bf16((x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6) * w).bfloat16(), ref, e32, "fp32 T5LayerNorm")
    bound = bf16_bound(ref, e32)
    out = ref.bfloat16()
    out[7, 4099] = _one_ulp_past(ref, bound, (7, 4099))
    with pytest.raises(AssertionError, match=r"worst at \(7, 4099\)"):
        check_bf16(out, ref, e32, "one element one ulp past")
    with pytest.raises(AssertionError):
        check_bf16(torch.roll(ref.bfloat16(), 1, dims=0), ref, e32, "rows shifted by one")
    with pytest.raises(AssertionError):
        check_bf16(torch.roll(ref.bfloat16(), 4, dims=1), ref, e32, "one float4 shifted")


def test_bitwise_checker_names_the_first_difference():
    a = torch.randn(5, 64).bfloat16()
    check_equal(a.clone(), a, "same")
    b = a.clone()
    b.view(torch.int16)[3, 9] ^= 1
    with pytest.raises(AssertionError, match=r"first at \(3, 9\)"):
        check_equal(b, a, "one bit")
    with pytest.raises(AssertionError):
        check_equal(torch.roll(a, 1, dims=0), a, "rows shifted by one")
    z = torch.zeros(4)
    with pytest.raises(AssertionError):     # -0.0 == 0.0, but not bit for bit
        check_equal(-z, z, "signed zero")


# ---------------------------------------------------------------------------------------------------------------------
# exact GEMM operand-form probes (pf_gemm_bf16 / pf_gemm_fp8)
# ---------------------------------------------------------------------------------------------------------------------
PROBE_MAX = 2                # |a|, |w| <= 2; bias, resid integers <= 16, gate <= 2


def probe_ints(shape, seed: int, device="cpu", lim: int = PROBE_MAX) -> torch.Tensor:
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randint(-lim, lim + 1, shape, generator=g, device=device).float()


def probe_exact(a: torch.Tensor, w: torch.Tensor, bias=None) -> torch.Tensor:
    """A W^T + bias in fp64 on integer operands, with a check that no partial sum can reach 2^24: then every fp32
    accumulation order gives this value exactly."""
    s = a.double() @ w.double().t()
    mag = a.double().abs() @ w.double().abs().t()
    if bias is not None:
        s = s + bias.double()
        mag = mag + bias.double().abs()
    assert float(mag.max()) < 2 ** 24
    return s


def fp8_slice_partials_ok(a: torch.Tensor, w: torch.Tensor, limit: float = 2 ** 11) -> bool:
    """Every 128-wide K slice of sum |a| |w| below `limit`.  The fp8 kernel adds each slice's wgmma partial into fp32
    (pf_b200.h FP8 contract); the partial itself comes from an accumulator of reduced precision, assumed exact for integers
    below 2^11.  That assumption has not been measured."""
    k = a.shape[-1]
    for k0 in range(0, k, 128):
        part = a[..., k0:k0 + 128].double().abs() @ w[:, k0:k0 + 128].double().abs().t()
        if float(part.max()) >= limit:
            return False
    return True


def gelu_tanh64(x):
    """0.5 x (1 + tanh(z)) (B:73-75) as x sigmoid(2 z): the same function, without the cancellation of 1 + tanh(z) that
    leaves no correct digit in fp64 for x below about -6."""
    x = x.double()
    return x * torch.sigmoid(2 * math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3))


def test_probe_operands_are_exact_in_any_fp32_order():
    a = probe_ints((300, 1000), 0).bfloat16()
    w = probe_ints((192, 1000), 1).bfloat16()
    bias = probe_ints((192,), 2, lim=16)
    exact = probe_exact(a, w, bias)
    assert torch.equal((a.float() @ w.float().t() + bias).double(), exact)
    assert torch.equal((a.float().flip(-1) @ w.float().flip(-1).t() + bias).double(), exact)
    # a column read from the neighbouring slice changes an integer
    neighbour = torch.cat([a[:, 1:], probe_ints((300, 1), 3).bfloat16()], 1)
    assert not torch.equal(probe_exact(neighbour, w, bias), exact)
    a8, w8 = probe_ints((64, 512), 4).to(torch.float8_e4m3fn), probe_ints((128, 512), 5).to(torch.float8_e4m3fn)
    assert torch.equal(a8.float(), probe_ints((64, 512), 4)) and fp8_slice_partials_ok(a8.float(), w8.float())
    assert not fp8_slice_partials_ok(torch.full((1, 128), 4.0), torch.full((1, 128), 4.0))


# ---------------------------------------------------------------------------------------------------------------------
# host-side argument checks: refused before any launch
# ---------------------------------------------------------------------------------------------------------------------
def test_row_kernel_entries_refuse_bad_arguments_without_a_launch():
    """Every pointer is a dummy that is never dereferenced: each call must be refused by an argument check, name the
    argument, and launch nothing."""
    lib = _lib.load()
    X, Y, S1, S2, W, R = 0x100000, 0x200000, 0x300000, 0x400000, 0x500000, 0x600000
    launches = lib.pf_launch_count()

    def refused(entry, args, what):
        rc = entry(*args)
        msg = lib.pf_last_error().decode()
        assert rc < 0 and what in msg, (entry.__name__, what, rc, msg)

    ln = (X, Y, 2, 16, 0, 16, 256, S1, S2, 1024, 1e-6, None)
    for i, arg, off in ((0, "x", 4), (7, "shift", 8), (8, "scale", 4), (1, "y", 4)):
        bad = list(ln)
        bad[i] += off
        refused(lib.pf_ln_modulate, bad, f"pf_ln_modulate: {arg} must be")
    ln8 = (X, Y, R, 2, 16, 0, 16, 256, S1, S2, 1024, 1e-6, None)
    for i, arg, off in ((0, "x", 8), (8, "shift", 4), (9, "scale", 12), (1, "y", 2), (2, "row_scale", 2)):
        bad = list(ln8)
        bad[i] += off
        refused(lib.pf_ln_modulate_fp8, bad, f"pf_ln_modulate_fp8: {arg} must be")

    rms = (X, Y, W, 2, 16, 0, 16, 4096, 1e-6, None)
    for i, arg, off in ((0, "x", 8), (2, "w", 4), (1, "y", 4)):
        bad = list(rms)
        bad[i] += off
        refused(lib.pf_rms_norm_rows, bad, f"pf_rms_norm_rows: {arg} must be")

    sl = [X, 2, 1920, W, S1, 5000, Y, 1, 0, 0, 0, None]
    refused(lib.pf_small_linear, sl[:3] + [W + 8] + sl[4:], "pf_small_linear: w must be")
    refused(lib.pf_small_linear, sl[:5] + [0] + sl[6:], "n=0")
    refused(lib.pf_small_linear, sl[:5] + [-8] + sl[6:], "n=-8")
    refused(lib.pf_small_linear, sl[:1] + [8, 1 << 28] + sl[3:], "too large")     # m k 4 = 2^33 wraps a 32-bit int

    pat = [X, 1, 2, 16, 3, 8, 12, Y, 100, 0, None]                 # b, c, t, h, w = 2, 16, 3, 8, 12
    for i, arg in ((2, "b"), (3, "c"), (4, "t")):
        bad = list(pat)
        bad[i] = 0
        refused(lib.pf_patchify, bad, f"{arg}=0")
    unp = [X, 100, 10, 2, 16, 3, 8, 12, Y, 1, None]                # rows [10, 10 + 3 * 4 * 6) of 100
    for i, arg in ((3, "b"), (4, "c"), (5, "t")):
        bad = list(unp)
        bad[i] = 0
        refused(lib.pf_unpatchify, bad, f"{arg}=0")
    refused(lib.pf_unpatchify, unp[:2] + [-1] + unp[3:], "row_begin=-1")
    refused(lib.pf_unpatchify, unp[:1] + [81] + unp[2:], "exceeds rows_per_batch 81")
    refused(lib.pf_unpatchify, unp[:2] + [29] + unp[3:], "exceeds rows_per_batch")
    assert lib.pf_launch_count() == launches
