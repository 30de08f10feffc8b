"""Per-element parity of the DiT and text-encoder row kernels on an H100, through the C ABI: LN + AdaLN modulate, the
small-M linear, the timestep sinusoid, patchify / unpatchify, CFG + Euler, the T5 RMSNorm rows and the token embedding
against the fp64 references and bounds of tests/test_row_kernels_cpu.py, and exact probes of the GEMM operand forms the
models use (bias NULL, A as a column slice, a gate shared across batches, QKV without RoPE, the FP8 path's A slices).
Output buffers start out holding a sentinel, so what a kernel must not write is checked too."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_row_kernels_cpu import (LIB_ULP, MUFU_REL, TIMESTEPS, U, cfg_euler_ref, check_bf16, check_bound, check_equal,
                                        fp8_slice_partials_ok, gamma, gelu_tanh64, ln_modulate_ref, ln_rows, probe_exact, probe_ints,
                                        rms_norm_ref, small_linear_ref, timestep_ref)

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = 7.5
TAIL = 64          # sentinel elements past the end of an output


def _lib():
    from pyramid_flow_b200 import _lib
    _lib.require_device()
    return _lib


def _buffer(n: int, dtype) -> torch.Tensor:
    """n elements followed by TAIL more, all SENTINEL."""
    return torch.full((n + TAIL,), SENTINEL, device=DEV, dtype=dtype)


def _tail_intact(buf: torch.Tensor, what: str) -> None:
    assert bool((buf[-TAIL:] == SENTINEL).all()), f"{what}: wrote past the end"


# ---------------------------------------------------------------------------------------------------------------------
# pf_ln_modulate
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [128, 768, 1280, 1536, 1920, 2048])
@pytest.mark.parametrize("batches", [1, 2, 3])
def test_ln_modulate(dim, batches):
    """The joint step's form (joint_step.py ln): shift / scale are column slices of the all-layer modulation rows, stride
    6 dim per batch; rows [r0, r0 + rc) of each batch.  Rows with |mean| / std up to 1e3 and 1e4 outliers; one constant
    row per batch, whose output is the shift exactly."""
    from pyramid_flow_b200 import ops
    S, r0, rc, eps = 45, 7, 30, 1e-6
    x = torch.stack([ln_rows(S, dim, 100 * dim + b, device=DEV) for b in range(batches)])
    const = torch.tensor([2.5, -3.25, 0.375][:batches], device=DEV)   # n c is exact in fp32: the row's deviations are 0
    x[:, r0 + 1] = const[:, None]
    g = torch.Generator(device=DEV).manual_seed(dim + batches)
    nm = 6 * dim
    mod = torch.randn(batches, nm, device=DEV, generator=g) * 0.5
    osh, osc = 3 * dim, 4 * dim
    y = torch.full((batches, S, dim), SENTINEL, device=DEV, dtype=torch.bfloat16)
    ops.ln_modulate(x, y, mod[:, osh:], mod[:, osc:], nm, batches=batches, rows_per_batch=S, row_begin=r0, row_count=rc, eps=eps)
    torch.cuda.synchronize()
    shift, scale = mod[:, None, osh:osh + dim], mod[:, None, osc:osc + dim]
    ref, e32 = ln_modulate_ref(x[:, r0:r0 + rc], shift, scale, eps)
    check_bf16(y[:, r0:r0 + rc], ref, e32, f"ln_modulate dim {dim}")
    check_equal(y[:, r0 + 1], shift[:, 0].bfloat16(), "constant row")
    assert bool((y[:, :r0] == SENTINEL).all()) and bool((y[:, r0 + rc:] == SENTINEL).all())


@pytest.mark.parametrize("dim", [768, 1280])
def test_ln_modulate_clip_layernorm(dim):
    """CLIP's LayerNorm as the text encoder runs it: mod_batch_stride 0, shift = bias, scale = weight - 1, eps 1e-5, against
    F.layer_norm with weight and bias in fp64.  Weights lie in [0.5, 2], where weight - 1 and 1 + (weight - 1) are exact
    in fp32, so the reference's weight is the kernel's 1 + scale."""
    from pyramid_flow_b200 import ops
    B, S, eps = 2, 77, 1e-5
    g = torch.Generator(device=DEV).manual_seed(dim)
    x = ln_rows(B * S, dim, dim, device=DEV).view(B, S, dim)
    weight = 0.5 + 1.5 * torch.rand(dim, device=DEV, generator=g)
    bias = torch.randn(dim, device=DEV, generator=g) * 0.2
    scale = weight - 1.0
    assert torch.equal(1.0 + scale, weight)
    y = torch.full((B, S, dim), SENTINEL, device=DEV, dtype=torch.bfloat16)
    ops.ln_modulate(x, y, bias, scale, 0, batches=B, rows_per_batch=S, row_begin=0, row_count=S, eps=eps)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.double(), (dim,), weight.double(), bias.double(), eps)
    _, e32 = ln_modulate_ref(x, bias, scale, eps)
    check_bf16(y, ref, e32, f"CLIP LayerNorm dim {dim}")


# ---------------------------------------------------------------------------------------------------------------------
# pf_small_linear
# ---------------------------------------------------------------------------------------------------------------------
FLAGS = [dict(), dict(bias=False), dict(act_in=1), dict(act_out=1), dict(accumulate=True), dict(round_in_bf16=True),
         dict(bias=False, act_in=1, act_out=1, accumulate=True, round_in_bf16=True)]


def _small_linear_case(m, k, n, flags, seed):
    lib = _lib().load()
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(m, k, device=DEV, generator=g) * 2
    w = (torch.randn(n, k, device=DEV, generator=g) / math.sqrt(k)).bfloat16()
    bias = torch.randn(n, device=DEV, generator=g) if flags.get("bias", True) else None
    acc = flags.get("accumulate", False)
    buf = _buffer(m * n, torch.float32)
    y0 = torch.randn(m, n, device=DEV, generator=g)
    if acc:
        buf[:m * n] = y0.view(-1)
    act_in, act_out, rnd = flags.get("act_in", 0), flags.get("act_out", 0), flags.get("round_in_bf16", False)
    rc = lib.pf_small_linear(x.data_ptr(), m, k, w.data_ptr(), None if bias is None else bias.data_ptr(), n, buf.data_ptr(),
                             act_in, act_out, int(acc), int(rnd), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.pf_last_error()
    torch.cuda.synchronize()
    ref, bound = small_linear_ref(x, w, bias, y0 if acc else None, act_in=act_in, act_out=act_out, round_in_bf16=rnd)
    check_bound(buf[:m * n].view(m, n), ref, bound, f"small_linear m {m} k {k} n {n} {flags}")
    _tail_intact(buf, "small_linear")


@pytest.mark.parametrize("m", range(1, 9))
def test_small_linear_every_instance(m):
    """Every template instance; k = 8, k not a multiple of 256, the > 48 KiB shared-memory path where m k 4 exceeds it, and
    the 96 KiB limit; n = 1 and n % 8 != 0; each flag alone and all together."""
    kmax = (96 * 1024 // (4 * m)) // 8 * 8
    shapes = [(8, 1), (264, 13), (1920, 77), (kmax, 9)]
    for i, (k, n) in enumerate(shapes):
        for j, flags in enumerate(FLAGS):
            _small_linear_case(m, k, n, flags, seed=1000 * m + 10 * i + j)


def test_small_linear_modulation_shape():
    """The per-step AdaLN modulation of every miniFLUX layer (joint_step.py: act_in SiLU, m = 2 CFG rows, k = 1920,
    n = (8 x 12 + 16 x 3 + 2) x 1920)."""
    m, k, n = 2, 1920, 146 * 1920
    lib = _lib().load()
    g = torch.Generator(device=DEV).manual_seed(7)
    x = torch.randn(m, k, device=DEV, generator=g)
    w = (torch.randn(n, k, device=DEV, generator=g) * 0.02).bfloat16()
    bias = torch.randn(n, device=DEV, generator=g) * 0.1
    buf = _buffer(m * n, torch.float32)
    assert lib.pf_small_linear(x.data_ptr(), m, k, w.data_ptr(), bias.data_ptr(), n, buf.data_ptr(), 1, 0, 0, 0,
                               torch.cuda.current_stream().cuda_stream) == 0, lib.pf_last_error()
    torch.cuda.synchronize()
    y = buf[:m * n].view(m, n)
    for c0 in range(0, n, 32768):
        c1 = min(n, c0 + 32768)
        ref, bound = small_linear_ref(x, w[c0:c1], bias[c0:c1], act_in=1)
        check_bound(y[:, c0:c1], ref, bound, f"modulation columns [{c0}, {c1})")
    _tail_intact(buf, "modulation")


# ---------------------------------------------------------------------------------------------------------------------
# pf_timestep_embedding
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [256, 2, 6, 258])
@pytest.mark.parametrize("round_bf16", [False, True])
def test_timestep_embedding(dim, round_bf16):
    lib = _lib().load()
    g = torch.Generator(device=DEV).manual_seed(dim)
    t = torch.cat([torch.tensor(TIMESTEPS, device=DEV), torch.rand(27, device=DEV, generator=g) * 1000])
    t = t.bfloat16().float()          # the caller's bf16 timesteps (P:750)
    m = t.numel()
    buf = _buffer(m * dim, torch.float32)
    assert lib.pf_timestep_embedding(t.data_ptr(), m, dim, buf.data_ptr(), int(round_bf16),
                                     torch.cuda.current_stream().cuda_stream) == 0, lib.pf_last_error()
    torch.cuda.synchronize()
    ref, bound = timestep_ref(t, dim, round_bf16)
    out = buf[:m * dim].view(m, dim)
    check_bound(out, ref, bound, f"timestep dim {dim}")
    if round_bf16:
        assert torch.equal(out, out.bfloat16().float())
    _tail_intact(buf, "timestep")


# ---------------------------------------------------------------------------------------------------------------------
# pf_patchify / pf_unpatchify: bitwise
# ---------------------------------------------------------------------------------------------------------------------
PATCH_SHAPES = [(3, 16, 1, 2, 2), (3, 16, 3, 8, 12), (1, 4, 5, 6, 10), (2, 16, 2, 10, 4)]   # b, c, t, h, w


@pytest.mark.parametrize("shape", PATCH_SHAPES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("tok_begin", [0, 10])
def test_patchify_unpatchify(shape, dtype, tok_begin):
    lib = _lib().load()
    stream = torch.cuda.current_stream().cuda_stream
    b, c, t, h, w = shape
    hh, ww, L, feat = h // 2, w // 2, t * (h // 2) * (w // 2), 4 * c
    rpb = tok_begin + L + 5                       # padding rows after the clip's tokens
    g = torch.Generator(device=DEV).manual_seed(sum(shape) + tok_begin)
    lat = torch.randn(shape, device=DEV, generator=g).to(dtype)
    tok = torch.full((b, rpb, feat), SENTINEL, device=DEV, dtype=torch.bfloat16)
    assert lib.pf_patchify(lat.data_ptr(), int(dtype == torch.float32), b, c, t, h, w, tok.data_ptr(), rpb, tok_begin,
                           stream) == 0, lib.pf_last_error()
    torch.cuda.synchronize()
    # F:285-286: b c t (h p1) (w p2) -> b (t h w) (p1 p2 c)
    want = lat.view(b, c, t, hh, 2, ww, 2).permute(0, 2, 3, 5, 4, 6, 1).reshape(b, L, feat).bfloat16()
    check_equal(tok[:, tok_begin:tok_begin + L], want, "patchify")
    assert bool((tok[:, :tok_begin] == SENTINEL).all()) and bool((tok[:, tok_begin + L:] == SENTINEL).all())

    x = torch.randn(b, rpb, feat, device=DEV, generator=g)        # every row distinct: a wrong row read shows
    for out_dtype in (torch.float32, torch.bfloat16):
        buf = _buffer(b * c * t * h * w, out_dtype)
        assert lib.pf_unpatchify(x.data_ptr(), rpb, tok_begin, b, c, t, h, w, buf.data_ptr(), int(out_dtype == torch.float32),
                                 stream) == 0, lib.pf_last_error()
        torch.cuda.synchronize()
        # F:383-387: b (t h w) (p1 p2 c) -> b c t (h p1) (w p2)
        want = x[:, tok_begin:tok_begin + L].reshape(b, t, hh, ww, 2, 2, c).permute(0, 6, 1, 2, 4, 3, 5).reshape(shape)
        check_equal(buf[:-TAIL].view(shape), want.to(out_dtype), f"unpatchify -> {out_dtype}")
        _tail_intact(buf, "unpatchify")


# ---------------------------------------------------------------------------------------------------------------------
# pf_cfg_euler_step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 1000, 4097])
def test_cfg_euler_step(n):
    lib = _lib().load()
    stream = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device=DEV).manual_seed(n)
    vu = torch.randn(n, device=DEV, generator=g)
    x = torch.randn(n, device=DEV, generator=g)

    def run(v2, guidance, dsigma):
        buf = _buffer(n, torch.float32)
        assert lib.pf_cfg_euler_step(v2.data_ptr(), guidance, dsigma, x.data_ptr(), buf.data_ptr(), n, stream) == 0
        torch.cuda.synchronize()
        _tail_intact(buf, "cfg_euler")
        return buf[:n]

    # exact cases: dsigma a power of two makes dsigma v exact, so x + dsigma v is one rounding in any evaluation; with
    # guidance 0, v = vu; with guidance 1 and vc / vu in [1/2, 2], vc - vu is exact (Sterbenz) and v = vc
    vc_near = vu * (0.6 + 1.2 * torch.rand(n, device=DEV, generator=g))
    v2 = torch.stack([vu, vc_near])
    check_equal(run(v2, 0.0, -0.0625), x + (-0.0625) * vu, "guidance 0")
    check_equal(run(v2, 1.0, -0.0625), x + (-0.0625) * vc_near, "guidance 1")
    v2 = torch.stack([vu, torch.randn(n, device=DEV, generator=g)])
    for guidance, dsigma in ((5.0, -0.05), (7.5, -0.0137), (1.0, 0.3)):
        ref, bound = cfg_euler_ref(v2, guidance, dsigma, x)
        check_bound(run(v2, guidance, dsigma), ref, bound, f"cfg_euler g {guidance}")


# ---------------------------------------------------------------------------------------------------------------------
# pf_rms_norm_rows, pf_embed_tokens
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [4, 100, 4096, 4100])
def test_rms_norm_rows(dim):
    """T5LayerNorm on rows [3, 16) of each of two batches; 100 has fewer float4s than lanes, 4100 one more than a lane
    sweep; rows scaled by 2^j; zero rows give zeros."""
    from pyramid_flow_b200 import ops
    B, S, r0, rc, eps = 2, 19, 3, 13, 1e-6
    g = torch.Generator(device=DEV).manual_seed(dim)
    x = torch.randn(B, S, dim, device=DEV, generator=g) * torch.exp2(torch.randint(-8, 9, (B, S, 1), device=DEV, generator=g).float())
    x[:, r0 + 2] = 0.0
    w = 1 + 0.3 * torch.randn(dim, device=DEV, generator=g)
    y = torch.full((B, S, dim), SENTINEL, device=DEV, dtype=torch.bfloat16)
    ops.rms_norm_rows(x, y, w, batches=B, rows_per_batch=S, row_begin=r0, row_count=rc, eps=eps)
    torch.cuda.synchronize()
    ref, e32 = rms_norm_ref(x[:, r0:r0 + rc], w, eps)
    check_bf16(y[:, r0:r0 + rc], ref, e32, f"rms_norm dim {dim}")
    assert bool((y[:, r0 + 2] == 0).all()), "zero row"      # 0 r w: the sign follows w
    assert bool((y[:, :r0] == SENTINEL).all()) and bool((y[:, r0 + rc:] == SENTINEL).all())


@pytest.mark.parametrize("dim", [4, 64])
def test_embed_tokens(dim):
    """ids 0 and vocab - 1, ids out of range (zero rows), the position table exactly rows_per_batch long; out =
    table[id] + pos[r % rows_per_batch] is one fp32 add of two bf16 values: the fp32 rounding of the fp64 sum, bit for bit."""
    lib = _lib().load()
    vocab, rpb, batches = 1000, 7, 3
    g = torch.Generator(device=DEV).manual_seed(dim)
    table = torch.randn(vocab, dim, device=DEV, generator=g).bfloat16()
    pos = (torch.randn(rpb, dim, device=DEV, generator=g) * 100).bfloat16()
    ids = torch.randint(0, vocab, (batches * rpb,), device=DEV, generator=g, dtype=torch.int32)
    ids[0], ids[rpb - 1], ids[rpb], ids[-1], ids[5] = 0, vocab - 1, vocab - 1, 0, -1
    ids[2 * rpb + 3] = vocab
    rows = ids.numel()
    valid = ((ids >= 0) & (ids < vocab))[:, None]
    base = torch.where(valid, table[ids.clamp(0, vocab - 1).long()].double(), 0.0)
    for pt in (pos, None):
        buf = _buffer(rows * dim, torch.float32)
        assert lib.pf_embed_tokens(ids.data_ptr(), rows, rpb, table.data_ptr(), vocab, dim, None if pt is None else pt.data_ptr(),
                                   rpb, buf.data_ptr(), torch.cuda.current_stream().cuda_stream) == 0, lib.pf_last_error()
        torch.cuda.synchronize()
        want = base if pt is None else torch.where(valid, base + pt.double().repeat(batches, 1), 0.0)
        check_equal(buf[:-TAIL].view(rows, dim), want.float(), f"embed_tokens pos {pt is not None}")
        _tail_intact(buf, "embed_tokens")


# ---------------------------------------------------------------------------------------------------------------------
# exact GEMM operand-form probes
# ---------------------------------------------------------------------------------------------------------------------
ACT_FLOOR = 2.0 ** -116      # approximate MUFU results below 2^-126 are flushed (.ftz), then scaled by |x| < 2^10


def _act_ref(epi, s):
    """(ref, e32) of the bf16-output activations on the exact sum s (fp64), e32 from the kernels' formulas
    (pf_common.cuh gelu_tanh_f, pf_gemm.cu epi_act)."""
    from pyramid_flow_b200._lib import PF_EPI_GELU_BF16, PF_EPI_GELU_ERF_BF16, PF_EPI_QUICK_GELU_BF16
    # x sigma(z) with sigma = 1 / (1 + 2^nu): a relative error d in 2^nu moves sigma by d (1 - sigma) relative.  nu is formed
    # from rounded constants and products, about 4u |nu| absolute; ex2 and rcp MUFU_REL each; 1 + 2^nu and x sigma u each
    if epi == PF_EPI_GELU_BF16:
        ref = gelu_tanh64(s)
        nu = 2 * math.sqrt(2 / math.pi) * math.log2(math.e) * (s.abs() + 0.044715 * s.abs() ** 3)
        sig = torch.sigmoid(2 * math.sqrt(2 / math.pi) * (s + 0.044715 * s ** 3))
        return ref, ref.abs() * (2 * MUFU_REL + 2 * U + 4 * U * nu * (1 - sig)) + ACT_FLOOR
    if epi == PF_EPI_QUICK_GELU_BF16:
        sig = torch.sigmoid(1.702 * s)
        ref = s * sig
        return ref, ref.abs() * (2 * MUFU_REL + 2 * U + 3 * 1.702 * U * s.abs() * (1 - sig)) + ACT_FLOOR
    assert epi == PF_EPI_GELU_ERF_BF16
    ref = 0.5 * s * (1 + torch.erf(s / math.sqrt(2)))
    # erff: LIB_ULP ulps of a result <= 1; its argument x / sqrt 2 rounded (erf' = 2 / sqrt(pi) exp(-x^2 / 2)); 1 + erf, the
    # products
    darg = 0.8 * U * s.abs() * torch.exp(-s * s / 2)
    return ref, 0.5 * s.abs() * (2 * LIB_ULP * U + 2 * U + darg) + 3 * U * ref.abs()


GEMM_B, GEMM_S, GEMM_R0, GEMM_RC = 2, 300, 40, 200


def _probe_a(k, off, seed):
    """A = x[..., off:off + k] of x [B, S, off + k + 24] whose other columns hold other integers."""
    x = probe_ints((GEMM_B, GEMM_S, off + k + 24), seed, device=DEV).bfloat16()
    return x[..., off:off + k]


@pytest.mark.parametrize("variant", [0, 1, 2])
@pytest.mark.parametrize("off", [0, 8])
def test_gemm_probe_plain_epilogues(variant, off):
    """Integer operands, k = 200 (not a multiple of the 64-wide K box), A a column slice (lda > k, offset off), bias NULL
    and integer: STORE_BF16 / STORE_F32 equal the exact result's RNE rounding bit for bit, the activations stay within
    their derived bounds; GEGLU on the 128-wide kernels."""
    from pyramid_flow_b200 import ops
    from pyramid_flow_b200._lib import (PF_EPI_GEGLU_BF16, PF_EPI_GELU_BF16, PF_EPI_GELU_ERF_BF16, PF_EPI_QUICK_GELU_BF16,
                                        PF_EPI_STORE_BF16, PF_EPI_STORE_F32)
    _lib()
    k, n = 200, 256
    a = _probe_a(k, off, 10 + off)
    w = probe_ints((n, k), 11, device=DEV).bfloat16()
    rows = dict(batches=GEMM_B, rows_per_batch=GEMM_S, row_begin=GEMM_R0, row_count=GEMM_RC, kernel_variant=variant)
    sl = slice(GEMM_R0, GEMM_R0 + GEMM_RC)
    for bias in (None, probe_ints((n,), 12, device=DEV, lim=16)):
        exact = probe_exact(a[:, sl], w, bias)
        for epi, dtype in ((PF_EPI_STORE_BF16, torch.bfloat16), (PF_EPI_STORE_F32, torch.float32), (PF_EPI_GELU_BF16, torch.bfloat16),
                           (PF_EPI_QUICK_GELU_BF16, torch.bfloat16), (PF_EPI_GELU_ERF_BF16, torch.bfloat16),
                           (PF_EPI_GEGLU_BF16, torch.bfloat16)):
            if epi == PF_EPI_GEGLU_BF16 and variant == 2:
                continue
            width = n // 2 if epi == PF_EPI_GEGLU_BF16 else n
            out = torch.full((GEMM_B, GEMM_S, width), SENTINEL, device=DEV, dtype=dtype)
            ops.gemm(a, w, bias, epi, out=out, **rows)
            torch.cuda.synchronize()
            what = f"epilogue {epi} variant {variant} off {off} bias {bias is not None}"
            got = out[:, sl]
            if epi in (PF_EPI_STORE_BF16, PF_EPI_STORE_F32):
                check_equal(got, exact.float().to(dtype), what)
            elif epi == PF_EPI_GEGLU_BF16:
                t = exact.view(GEMM_B, GEMM_RC, n // 128, 2, 64)
                gate, lin = t[:, :, :, 0], t[:, :, :, 1]
                gref, ge = _act_ref(PF_EPI_GELU_BF16, gate)
                ref = (gref * lin).reshape(GEMM_B, GEMM_RC, width)
                check_bf16(got, ref, ((ge * lin.abs()).reshape_as(ref) + U * ref.abs()), what)
            else:
                ref, e32 = _act_ref(epi, exact)
                check_bf16(got, ref, e32, what)
            assert bool((out[:, :GEMM_R0] == SENTINEL).all()) and bool((out[:, GEMM_R0 + GEMM_RC:] == SENTINEL).all()), what


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_gemm_probe_gate_resid(variant):
    """GATE_RESID on an A column slice, bias NULL and integer, the gate per batch and shared (gate_batch_stride 0, the
    text encoders' ones gate and the x-embedder gate), on both residual read-modify-write paths: bit for bit."""
    from pyramid_flow_b200 import _lib as L, ops
    from pyramid_flow_b200._lib import PF_EPI_GATE_RESID, PF_OPT_GEMM_STAGED_RESID
    _lib()
    k, n = 200, 256
    a = _probe_a(k, 8, 20)
    w = probe_ints((n, k), 21, device=DEV).bfloat16()
    resid0 = probe_ints((GEMM_B, GEMM_S, n), 22, device=DEV, lim=16)
    rows = dict(batches=GEMM_B, rows_per_batch=GEMM_S, row_begin=GEMM_R0, row_count=GEMM_RC, kernel_variant=variant)
    sl = slice(GEMM_R0, GEMM_R0 + GEMM_RC)
    saved = L.get_option(PF_OPT_GEMM_STAGED_RESID)
    try:
        for staged in (0, 1):
            L.set_option(PF_OPT_GEMM_STAGED_RESID, staged)
            for bias in (None, probe_ints((n,), 23, device=DEV, lim=16)):
                exact = probe_exact(a[:, sl], w, bias)
                for shared in (False, True):
                    gate = probe_ints((n,) if shared else (GEMM_B, n), 24 + shared, device=DEV)
                    out = resid0.clone()
                    ops.gemm(a, w, bias, PF_EPI_GATE_RESID, out=out, gate=gate, gate_batch_stride=0 if shared else n, **rows)
                    torch.cuda.synchronize()
                    gb = gate[None, None] if shared else gate[:, None]
                    want = (resid0[:, sl].double() + gb.double() * exact).float()
                    what = f"GATE_RESID variant {variant} staged {staged} bias {bias is not None} shared gate {shared}"
                    check_equal(out[:, sl], want, what)
                    assert torch.equal(out[:, :GEMM_R0], resid0[:, :GEMM_R0]), what
                    assert torch.equal(out[:, GEMM_R0 + GEMM_RC:], resid0[:, GEMM_R0 + GEMM_RC:]), what
    finally:
        L.set_option(PF_OPT_GEMM_STAGED_RESID, saved)


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_gemm_probe_qkv_without_rope(variant):
    """QKV_ROPE with rope NULL and bias NULL / integer on an A column slice: v is the exact sum rounded once (bit for bit),
    q and k its per-head RMSNorm (fp32 sum of squares, rsqrtf, two products) within the derived bound."""
    from pyramid_flow_b200 import ops
    from pyramid_flow_b200._lib import PF_EPI_QKV_ROPE
    _lib()
    H, hd, k = 2, 64, 200
    n = 3 * H * hd
    a = _probe_a(k, 8, 30)
    w = probe_ints((n, k), 31, device=DEV).bfloat16()
    g = torch.Generator(device=DEV).manual_seed(32)
    qn, kn = 0.5 + torch.rand(hd, device=DEV, generator=g), 0.5 + torch.rand(hd, device=DEV, generator=g)
    sl = slice(GEMM_R0, GEMM_R0 + GEMM_RC)
    eps = 1e-6
    for bias in (None, probe_ints((n,), 33, device=DEV, lim=16)):
        outs = [torch.full((GEMM_B, H, GEMM_S, hd), SENTINEL, device=DEV, dtype=torch.bfloat16) for _ in range(3)]
        ops.gemm(a, w, bias, PF_EPI_QKV_ROPE, batches=GEMM_B, rows_per_batch=GEMM_S, row_begin=GEMM_R0, row_count=GEMM_RC,
                 q_out=outs[0], k_out=outs[1], v_out=outs[2], rope=None, q_norm_w=qn, k_norm_w=kn, norm_eps=eps, heads=H,
                 head_dim=hd, seq_len=GEMM_S, kernel_variant=variant)
        torch.cuda.synchronize()
        exact = probe_exact(a[:, sl], w, bias).view(GEMM_B, GEMM_RC, 3, H, hd).permute(2, 0, 3, 1, 4)   # [3, B, H, rc, hd]
        what = f"QKV variant {variant} bias {bias is not None}"
        check_equal(outs[2][:, :, sl], exact[2].float().bfloat16(), what + " v")
        for j, nw in ((0, qn), (1, kn)):
            s = exact[j]
            ref = s * nw.double() / torch.sqrt((s * s).mean(-1, keepdim=True) + eps)
            check_bf16(outs[j][:, :, sl], ref, ref.abs() * (0.5 * gamma(66) + 2 * LIB_ULP * U + 4 * U), f"{what} {'qk'[j]}")
        for o in outs:
            assert bool((o[:, :, :GEMM_R0] == SENTINEL).all()) and bool((o[:, :, GEMM_R0 + GEMM_RC:] == SENTINEL).all()), what


def test_gemm_fp8_probe_a_slices():
    """pf_gemm_fp8 on the two A slices of the FP8 joint step (xn8[:, :, :wa] for the attention output projection,
    xn8[:, :, wa:] for the MLP down projection): e4m3 integers with power-of-two row and column scales, so the dequantised
    result is exact; every 128-wide K slice's partial stays below 2^11, where the fp8 accumulator is assumed exact.
    STORE_F32 and GATE_RESID, bias NULL and integer: bit for bit."""
    from pyramid_flow_b200 import ops
    from pyramid_flow_b200._lib import PF_EPI_GATE_RESID, PF_EPI_STORE_F32
    _lib()
    wa, wf, n = 256, 384, 256
    xi = probe_ints((GEMM_B, GEMM_S, wa + wf), 40, device=DEV)
    x8 = xi.to(torch.float8_e4m3fn)
    assert torch.equal(x8.float(), xi)
    g = torch.Generator(device=DEV).manual_seed(41)
    a_scale = torch.exp2(torch.randint(-2, 3, (GEMM_B, GEMM_S), device=DEV, generator=g).float())
    w_scale = torch.exp2(torch.randint(-2, 3, (n,), device=DEV, generator=g).float())
    resid0 = probe_ints((GEMM_B, GEMM_S, n), 42, device=DEV, lim=16)
    gate = probe_ints((GEMM_B, n), 43, device=DEV)
    rows = dict(batches=GEMM_B, rows_per_batch=GEMM_S, row_begin=GEMM_R0, row_count=GEMM_RC)
    sl = slice(GEMM_R0, GEMM_R0 + GEMM_RC)
    for c0, c1, seed in ((0, wa, 44), (wa, wa + wf, 45)):
        a8 = x8[:, :, c0:c1]
        wi = probe_ints((n, c1 - c0), seed, device=DEV)
        w8 = wi.to(torch.float8_e4m3fn)
        assert fp8_slice_partials_ok(xi[:, sl, c0:c1], wi)
        for bias in (None, probe_ints((n,), seed + 10, device=DEV, lim=16)):
            acc = probe_exact(xi[:, sl, c0:c1], wi) * a_scale[:, sl, None].double() * w_scale.double()
            y = acc if bias is None else acc + bias.double()
            what = f"fp8 A[:, :, {c0}:{c1}] bias {bias is not None}"
            out = torch.full((GEMM_B, GEMM_S, n), SENTINEL, device=DEV)
            ops.gemm_fp8(a8, a_scale, w8, w_scale, bias, PF_EPI_STORE_F32, out=out, **rows)
            res = resid0.clone()
            ops.gemm_fp8(a8, a_scale, w8, w_scale, bias, PF_EPI_GATE_RESID, out=res, gate=gate, gate_batch_stride=n, **rows)
            torch.cuda.synchronize()
            check_equal(out[:, sl], y.float(), what + " STORE_F32")
            assert bool((out[:, :GEMM_R0] == SENTINEL).all()) and bool((out[:, GEMM_R0 + GEMM_RC:] == SENTINEL).all()), what
            check_equal(res[:, sl], (resid0[:, sl].double() + gate[:, None].double() * y).float(), what + " GATE_RESID")
            assert torch.equal(res[:, :GEMM_R0], resid0[:, :GEMM_R0]), what
