"""Per-kernel parity through the C-ABI on an H100 (ragged shapes included): GEMM epilogues, attention mask cases,
elementwise kernels.  The checker for a single floating-point kernel is a plain PyTorch fp32 reference of the same op."""
import pytest
import os

import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-20)).item()


@pytest.mark.parametrize("m,n,k", [(128, 64, 64), (1, 64, 64), (129, 256, 128), (300, 1920, 1920), (1000, 192, 512),
                                   (777, 128, 4096), (2048, 1920, 9600), (5, 7680, 1920)])
def test_gemm_bias_store(m, n, k):
    from pyramid_flow_b200 import ops
    torch.manual_seed(m * 7 + n)
    x = (torch.randn(m, k, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(n, k, device=DEV) * 0.05).bfloat16()
    b = torch.randn(n, device=DEV)
    y = ops.linear_bf16(x, w, b)
    torch.cuda.synchronize()
    assert _rel(y, x.float() @ w.float().t() + b) < 8e-3      # bf16 output rounding: 2^-8 relative


def test_gemm_rejects_bad_shapes():
    from pyramid_flow_b200 import ops
    x = torch.zeros(8, 60, device=DEV, dtype=torch.bfloat16)      # K not a multiple of 8 elements / N not a multiple of 64
    w = torch.zeros(100, 60, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        ops.linear_bf16(x, w, None)


def test_gemm_epilogues_row_ranges():
    from pyramid_flow_b200 import ops
    from pyramid_flow_b200._lib import PF_EPI_GATE_RESID, PF_EPI_GELU_BF16, PF_EPI_QKV_GELU, PF_EPI_QKV_ROPE, PF_EPI_STORE_F32
    torch.manual_seed(1)
    B, S, D, H, T0, hd = 2, 300, 384, 6, 40, 64
    x = (torch.randn(B, S, D, device=DEV) * 0.5).bfloat16()
    w = (torch.randn(4 * D, D, device=DEV) * 0.05).bfloat16()
    bias = torch.randn(4 * D, device=DEV) * 0.1
    out = torch.zeros(B, S, 4 * D, device=DEV, dtype=torch.bfloat16)
    ops.gemm(x, w, bias, PF_EPI_GELU_BF16, batches=B, rows_per_batch=S, row_begin=T0, row_count=S - T0, out=out)
    ref = F.gelu(x[:, T0:].float() @ w.float().t() + bias, approximate="tanh")
    assert _rel(out[:, T0:], ref) < 8e-3 and bool((out[:, :T0] == 0).all())
    w2 = (torch.randn(D, D, device=DEV) * 0.05).bfloat16()
    b2 = torch.randn(D, device=DEV) * 0.1
    o32 = torch.zeros(B, S, D, device=DEV)
    ops.gemm(x, w2, b2, PF_EPI_STORE_F32, batches=B, rows_per_batch=S, row_begin=0, row_count=T0, out=o32)
    assert _rel(o32[:, :T0], x[:, :T0].float() @ w2.float().t() + b2) < 1e-5 and bool((o32[:, T0:] == 0).all())
    resid = torch.randn(B, S, D, device=DEV)
    r0 = resid.clone()
    gate = torch.randn(B, 3 * D, device=DEV)
    ops.gemm(x, w2, b2, PF_EPI_GATE_RESID, batches=B, rows_per_batch=S, row_begin=T0, row_count=S - T0, out=resid,
             gate=gate[:, D:], gate_batch_stride=3 * D)
    ref = r0[:, T0:] + gate[:, None, D:2 * D] * (x[:, T0:].float() @ w2.float().t() + b2)
    assert _rel(resid[:, T0:], ref) < 1e-5 and bool((resid[:, :T0] == r0[:, :T0]).all())
    # QKV: bias + per-head RMSNorm + RoPE, head-major stores
    wq = (torch.randn(3 * D, D, device=DEV) * 0.05).bfloat16()
    bq = torch.randn(3 * D, device=DEV) * 0.1
    qn, kn = 1 + 0.1 * torch.randn(hd, device=DEV), 1 + 0.1 * torch.randn(hd, device=DEV)
    ang = torch.randn(S, hd // 2, device=DEV)
    rope = torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous()

    def ref_qkv(xr, pos0):
        y = xr.float() @ wq.float().t() + bq
        qq, kk, vv = y.chunk(3, dim=-1)
        n = xr.shape[1]

        def nr(t, wn):
            t = t.view(B, n, H, hd)
            t = t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6) * wn
            c, s_ = rope[pos0:pos0 + n, :, 0][None, :, None, :], rope[pos0:pos0 + n, :, 1][None, :, None, :]
            t2 = t.view(B, n, H, hd // 2, 2)
            return torch.stack([c * t2[..., 0] - s_ * t2[..., 1], s_ * t2[..., 0] + c * t2[..., 1]], -1).view(B, n, H, hd).transpose(1, 2)
        return nr(qq, qn), nr(kk, kn), vv.view(B, n, H, hd).transpose(1, 2)

    qo = torch.zeros(B, H, S, hd, device=DEV, dtype=torch.bfloat16)
    ko, vo = torch.zeros_like(qo), torch.zeros_like(qo)
    ops.gemm(x, wq, bq, PF_EPI_QKV_ROPE, batches=B, rows_per_batch=S, row_begin=T0, row_count=S - T0, q_out=qo, k_out=ko,
             v_out=vo, rope=rope, q_norm_w=qn, k_norm_w=kn, heads=H, head_dim=hd, seq_len=S)
    rq, rk, rv = ref_qkv(x[:, T0:], T0)
    assert _rel(qo[:, :, T0:], rq) < 8e-3 and _rel(ko[:, :, T0:], rk) < 8e-3 and _rel(vo[:, :, T0:], rv) < 8e-3
    assert bool((qo[:, :, :T0] == 0).all())
    wm = (torch.randn(4 * D, D, device=DEV) * 0.05).bfloat16()
    bm = torch.randn(4 * D, device=DEV) * 0.1
    cat = torch.zeros(B, S, 5 * D, device=DEV, dtype=torch.bfloat16)
    ops.gemm(x, torch.cat([wq, wm], 0).contiguous(), torch.cat([bq, bm], 0).contiguous(), PF_EPI_QKV_GELU, batches=B,
             rows_per_batch=S, row_begin=0, row_count=S, out=cat, out_col_begin=D, q_out=qo, k_out=ko, v_out=vo, rope=rope,
             q_norm_w=qn, k_norm_w=kn, heads=H, head_dim=hd, seq_len=S, n_split=3 * D)
    rq, rk, rv = ref_qkv(x, 0)
    assert _rel(qo, rq) < 8e-3 and _rel(vo, rv) < 8e-3
    assert _rel(cat[..., D:], F.gelu(x.float() @ wm.float().t() + bm, approximate="tanh")) < 8e-3


# pf_attn_desc.variant: every accepted value (3, 0x10 with the pair schedule, 0x20 with the group schedule, 0 = default) must
# give the same, correct result; the sm_90a library runs one kernel for all of them
# PF_TEST_ATTN_EXTRA = further variant codes to put through the same cases
ATTN_EXTRA = [int(x, 0) for x in os.environ.get("PF_TEST_ATTN_EXTRA", "").split()]
ATTN_VARIANTS = [3, 0x10, 0x20, 0] + ATTN_EXTRA


def _attn_ref(q, k, v, sg, tm):
    B, H, S, _ = q.shape
    mask = (sg[:, :, None] == sg[:, None, :]) & (tm[:, :, None] >= tm[:, None, :])
    ref = F.scaled_dot_product_attention(q.float(), k.float(), v.float(), attn_mask=mask[:, None])
    return ref.transpose(1, 2).reshape(B, S, H * 64), mask


def _attn_case(B, H, S, seg, tim, scale_q=1.0):
    """max |out - fp32 SDPA(dense mask)| over every kernel variant; also q_row_begin (rows below it stay untouched)."""
    from pyramid_flow_b200 import ops
    q = (torch.randn(B, H, S, 64, device=DEV) * scale_q).bfloat16()
    k = torch.randn(B, H, S, 64, device=DEV).bfloat16()
    v = torch.randn(B, H, S, 64, device=DEV).bfloat16()
    sched, pairs = ops.attn_build_schedule(seg, tim)
    psched = ops.attn_build_pair_schedule(sched, S, seg, tim).to(DEV)
    sg, tm = seg.to(DEV).int(), tim.to(DEV).int()
    ref, mask = _attn_ref(q, k, v, sg, tm)
    assert int(pairs.sum()) == int(mask.sum())
    worst = 0.0
    for variant in ATTN_VARIANTS:
        out = torch.zeros(B, S, H * 64, device=DEV, dtype=torch.bfloat16)
        ops.attn_fwd(q, k, v, out, sg, tm, sched.to(DEV), 0.125, variant=variant, pair_sched=psched)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(out.float()).all()), variant
        worst = max(worst, (out.float() - ref).abs().max().item())
        for qb in sorted({((S - 1) // 128) * 128, (S // 256) * 128}):
            if qb == 0:
                continue
            o2 = torch.full((B, S, H * 64), 7.0, device=DEV, dtype=torch.bfloat16)
            ops.attn_fwd(q, k, v, o2, sg, tm, sched.to(DEV), 0.125, variant=variant, q_row_begin=qb, pair_sched=psched)
            torch.cuda.synchronize()
            assert torch.equal(o2[:, qb:], out[:, qb:]) and bool((o2[:, :qb] == 7.0).all()), (variant, qb)
    return worst


def test_attention_mask_cases():
    torch.manual_seed(3)
    # shorter than one tile; dense; tile-aligned causal; ragged text + frames not aligned to tiles; sequence tail
    assert _attn_case(1, 2, 77, torch.ones(1, 77, dtype=torch.int32), torch.zeros(1, 77, dtype=torch.int32)) < 2e-2
    assert _attn_case(1, 2, 256, torch.ones(1, 256, dtype=torch.int32), torch.zeros(1, 256, dtype=torch.int32)) < 2e-2
    tim = torch.cat([torch.zeros(128), torch.ones(128), 2 * torch.ones(128)]).int()[None]
    assert _attn_case(1, 2, 384, torch.ones(1, 384, dtype=torch.int32), tim) < 2e-2
    S = 128 + 60 * 5
    tim = torch.cat([torch.zeros(128 + 60)] + [torch.full((60,), i + 1.0) for i in range(4)]).int()[None].repeat(2, 1)
    seg = torch.ones(2, S, dtype=torch.int32)
    seg[0, 37:128] = 0
    assert _attn_case(2, 3, S, seg, tim) < 2e-2
    S = 77 + 240 * 9 + 13
    tim = torch.cat([torch.zeros(77 + 240)] + [torch.full((240,), i + 1.0) for i in range(8)] + [torch.full((13,), 9.0)]).int()[None].repeat(2, 1)
    seg = torch.ones(2, S, dtype=torch.int32)
    seg[1, 50:77] = 0
    assert _attn_case(2, 4, S, seg, tim) < 2e-2
    # long frames (q-tile pairs whose kv lists differ by many tiles), odd tile count
    S = 128 + 200 + 1000 + 1700
    tim = torch.cat([torch.zeros(128 + 200), torch.ones(1000), 2 * torch.ones(1700)]).int()[None].repeat(2, 1)
    seg = torch.ones(2, S, dtype=torch.int32)
    seg[0, 100:128] = 0
    assert _attn_case(2, 2, S, seg, tim) < 2e-2


def test_attention_adversarial_score_jumps():
    """Scores that jump by hundreds of log2 units between neighbouring kv tiles, rising and falling (the exponent argument must
    never overflow; rows dominated by one tile must come out exact), and a pair schedule consistent with the tile schedule."""
    from pyramid_flow_b200 import ops
    torch.manual_seed(11)
    B, H, S = 1, 2, 1024
    q = torch.randn(B, H, S, 64, device=DEV).bfloat16()
    k = torch.randn(B, H, S, 64, device=DEV)
    amp = torch.tensor([1.0, 60.0, 0.02, 250.0, 1.0, 0.001, 120.0, 5.0], device=DEV)       # per kv tile
    k = (k * amp.repeat_interleave(128)[None, None, :, None]).bfloat16()
    v = torch.randn(B, H, S, 64, device=DEV).bfloat16()
    seg = torch.ones(B, S, dtype=torch.int32)
    tim = (torch.arange(S) // 256).int()[None]
    sched, _ = ops.attn_build_schedule(seg, tim)
    pso = ops.attn_build_pair_schedule(sched, S, seg, tim)
    psched = pso.sched
    # pair rows: union of the two tiles' lists, flags consistent with the tile rows
    qt = S // 128
    for p in range((qt + 1) // 2):
        hi, lo = qt - 1 - 2 * p, qt - 2 - 2 * p
        n = int(psched[0, p, 0])
        ent = psched[0, p, 1:1 + n].tolist()
        for x, t in ((0, lo), (1, hi)):
            if t < 0:
                assert all(((e >> (2 * x)) & 3) == 0 for e in ent)
                continue
            own = [((e >> 4) << 1) | (((e >> (2 * x)) & 2) >> 1) for e in ent if (e >> (2 * x)) & 1]
            assert own == sched[0, t, 1:1 + int(sched[0, t, 0])].tolist()
    sg, tm = seg.to(DEV), tim.to(DEV)
    ref, _ = _attn_ref(q, k, v, sg, tm)
    # the online softmax keeps an exact per-row running max and must be exact on such inputs
    for variant in [0x10, 0x20, 0] + ATTN_EXTRA:
        out = torch.zeros(B, S, H * 64, device=DEV, dtype=torch.bfloat16)
        ops.attn_fwd(q, k, v, out, sg, tm, sched.to(DEV), 0.125, variant=variant, pair_sched=pso.to(DEV))
        torch.cuda.synchronize()
        assert bool(torch.isfinite(out.float()).all()), variant
        assert (out.float() - ref).abs().max().item() < 3e-2, variant


def test_elementwise_kernels():
    from einops import rearrange
    from pyramid_flow_b200 import ops
    torch.manual_seed(2)
    B, S, D = 2, 333, 1920
    x = torch.randn(B, S, D, device=DEV) * 2 + 0.3
    mod = torch.randn(B, 6 * D, device=DEV) * 0.3
    y = torch.zeros(B, S, D, device=DEV, dtype=torch.bfloat16)
    ops.ln_modulate(x, y, mod[:, 0:], mod[:, D:], 6 * D, batches=B, rows_per_batch=S, row_begin=77, row_count=S - 77)
    ref = F.layer_norm(x[:, 77:], (D,), eps=1e-6) * (1 + mod[:, None, D:2 * D]) + mod[:, None, :D]
    assert _rel(y[:, 77:], ref) < 8e-3 and bool((y[:, :77] == 0).all())
    xm = torch.randn(2, 1920, device=DEV)
    w = (torch.randn(5000, 1920, device=DEV) * 0.05).bfloat16()
    b = torch.randn(5000, device=DEV)
    yo = torch.zeros(2, 5000, device=DEV)
    ops.small_linear(xm, w, b, yo, act_in=1)
    ref = F.silu(xm) @ w.float().t() + b
    assert _rel(yo, ref) < 1e-5
    ops.small_linear(xm, w, b, yo, act_out=1, accumulate=True)
    assert _rel(yo, ref + F.silu(xm @ w.float().t() + b)) < 1e-5
    t = torch.tensor([972.0, 3.5], device=DEV)
    e = ops.timestep_embedding(t, 256, round_bf16=False)
    arg = t[:, None] * torch.exp(-torch.log(torch.tensor(10000.0)) * torch.arange(128, device=DEV).float() / 128)[None]
    assert (e - torch.cat([arg.cos(), arg.sin()], -1)).abs().max().item() < 2e-3     # |arg| ~ 1e3: fp32 sin/cos ulps
    lat = torch.randn(2, 16, 2, 8, 12, device=DEV).bfloat16()
    L = 2 * 4 * 6
    tok = torch.zeros(2, 10 + L, 64, device=DEV, dtype=torch.bfloat16)
    ops.patchify(lat, tok, 10 + L, 10)
    ref = rearrange(rearrange(lat, "b c t h w -> b t h w c"), "b t (h p1) (w p2) c -> b (t h w) (p1 p2 c)", p1=2, p2=2)
    assert bool((tok[:, 10:] == ref).all())                                           # byte/index work: bit-exact
    out = torch.zeros(2, 16, 2, 8, 12, device=DEV)
    ops.unpatchify(tok.float().contiguous(), 10 + L, 10, out)
    assert bool((out == lat.float()).all())
    v2, xs, xo = torch.randn(2, 1000, device=DEV), torch.randn(1000, device=DEV), torch.zeros(1000, device=DEV)
    ops.cfg_euler_step(v2, 5.0, -0.05, xs, xo)
    assert (xo - (xs + (-0.05) * (v2[0] + 5.0 * (v2[1] - v2[0])))).abs().max().item() < 1e-5


def test_step_context_record_and_replay():
    """pf_ctx (include/pf_b200.h): a launch sequence recorded once (LN+modulate -> GEMM+GELU -> gated-residual GEMM -> masked
    attention) and re-issued by pf_dit_step_flux(ctx) gives the same bits as the direct launches, on new input values."""
    import ctypes as C
    from pyramid_flow_b200 import _lib, ops
    from pyramid_flow_b200._lib import PF_EPI_GATE_RESID, PF_EPI_GELU_BF16
    lib = _lib.load()
    _lib.require_device()
    torch.manual_seed(5)
    B, S, D, H = 1, 384, 256, 4
    x = torch.randn(B, S, D, device=DEV)
    mod = torch.randn(B, 3 * D, device=DEV) * 0.3
    w1 = (torch.randn(4 * D, D, device=DEV) * 0.05).bfloat16()
    b1 = torch.randn(4 * D, device=DEV) * 0.1
    w2 = (torch.randn(D, 4 * D, device=DEV) * 0.05).bfloat16()
    b2 = torch.randn(D, device=DEV) * 0.1
    xn = torch.zeros(B, S, D, device=DEV, dtype=torch.bfloat16)
    hid = torch.zeros(B, S, 4 * D, device=DEV, dtype=torch.bfloat16)
    q = torch.randn(B, H, S, 64, device=DEV).bfloat16()
    k = torch.randn(B, H, S, 64, device=DEV).bfloat16()
    v = torch.randn(B, H, S, 64, device=DEV).bfloat16()
    att = torch.zeros(B, S, H * 64, device=DEV, dtype=torch.bfloat16)
    seg = torch.ones(B, S, dtype=torch.int32)
    tim = (torch.arange(S) // 128).int()[None]
    sched, _ = ops.attn_build_schedule(seg, tim)
    ps = ops.attn_build_pair_schedule(sched, S, seg, tim).to(DEV)
    sg, tm, sc = seg.to(DEV), tim.to(DEV), sched.to(DEV)

    def sequence():
        ops.ln_modulate(x, xn, mod[:, 0:], mod[:, D:], 3 * D, batches=B, rows_per_batch=S, row_begin=0, row_count=S)
        ops.gemm(xn, w1, b1, PF_EPI_GELU_BF16, batches=B, rows_per_batch=S, out=hid)
        ops.gemm(hid, w2, b2, PF_EPI_GATE_RESID, batches=B, rows_per_batch=S, out=x, ldo=D, gate=mod[:, 2 * D:], gate_batch_stride=3 * D)
        ops.attn_fwd(q, k, v, att, sg, tm, sc, 0.125, pair_sched=ps)

    x0 = x.clone()
    sequence()
    torch.cuda.synchronize()
    x_direct, att_direct = x.clone(), att.clone()
    ctx = C.c_void_p()
    _lib.check(lib.pf_ctx_create(C.byref(ctx)), "pf_ctx_create")
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        _lib.check(lib.pf_ctx_record_begin(ctx, side.cuda_stream), "pf_ctx_record_begin")
        sequence()                                  # recorded, not executed
        n = lib.pf_ctx_record_end(ctx)
    assert n >= 4, (n, lib.pf_last_error())
    torch.cuda.synchronize()
    assert torch.equal(x, x_direct), "recording must not execute the launches"
    x.copy_(x0)
    att.zero_()
    _lib.check(lib.pf_dit_step_flux(ctx, torch.cuda.current_stream().cuda_stream), "pf_dit_step_flux")
    torch.cuda.synchronize()
    assert torch.equal(x, x_direct) and torch.equal(att, att_direct)
    # new values in the same buffers: replay follows
    x.copy_(x0 * 0.5 + 0.1)
    q.copy_(torch.randn_like(q.float()).bfloat16())
    _lib.check(lib.pf_dit_step_flux(ctx, torch.cuda.current_stream().cuda_stream), "pf_dit_step_flux")
    torch.cuda.synchronize()
    x_rep, att_rep = x.clone(), att.clone()
    x.copy_(x0 * 0.5 + 0.1)
    sequence()
    torch.cuda.synchronize()
    assert torch.equal(x, x_rep) and torch.equal(att, att_rep)
    _lib.check(lib.pf_ctx_destroy(ctx), "pf_ctx_destroy")


def test_stage_hop_kernel():
    """pf_stage_hop == alpha * nearest_x2(x) + beta * (L z per 2x2 block) computed in torch on the same normals (P:729-743,
    P:697-703), and the block covariance of the generated noise is (1+gamma) I - gamma 11^T."""
    from einops import rearrange
    from pyramid_flow_b200 import ops
    torch.manual_seed(4)
    gamma, alpha, beta = 1.0 / 3.0, 0.74963, 0.43366
    for dtype in (torch.float32, torch.bfloat16):
        x = torch.randn(2, 16, 3, 12, 20, device=DEV).to(dtype)
        z = torch.randn(2, 16, 3, 24, 40, device=DEV)
        out = ops.stage_hop(x, z, alpha, beta, gamma)
        cov = torch.eye(4, dtype=torch.float64) * (1 + gamma) - torch.ones(4, 4, dtype=torch.float64) * gamma
        L = torch.linalg.cholesky(cov).float().to(DEV)
        zb = rearrange(z, "b c t (h p) (w q) -> (b c t h w) (p q)", p=2, q=2)
        nb = rearrange(zb @ L.T, "(b c t h w) (p q) -> b c t (h p) (w q)", b=2, c=16, t=3, h=12, w=20, p=2, q=2)
        up = torch.nn.functional.interpolate(x.float(), scale_factor=(1, 2, 2), mode="nearest")
        ref = alpha * up + beta * nb
        tol = 1e-5 if dtype == torch.float32 else 2e-2
        assert (out.float() - ref).abs().max().item() < tol
    xz = torch.zeros(1, 16, 8, 48, 80, device=DEV)
    n = ops.stage_hop(xz, torch.randn(1, 16, 8, 96, 160, device=DEV), 1.0, 1.0, gamma)
    blocks = rearrange(n, "b c t (h p) (w q) -> (b c t h w) (p q)", p=2, q=2).double()
    emp = blocks.T @ blocks / blocks.shape[0]
    assert (emp.cpu() - cov).abs().max().item() < 0.02


def test_gemm_library_options_do_not_change_bits():
    """pf_set_option data-path choices (GATE_RESID read-modify-write staged through shared memory; wave-quantisation-aware tile
    width) compute the same sums in the same order: outputs are bit-identical to the default path, for row ranges, ragged M
    and the sequence-parallel chunk shape (M=3872, N=1920) whose tiling actually changes."""
    from pyramid_flow_b200 import _lib, ops
    from pyramid_flow_b200._lib import (PF_EPI_GATE_RESID, PF_EPI_GELU_BF16, PF_EPI_STORE_BF16, PF_OPT_GEMM_STAGED_RESID,
                                        PF_OPT_GEMM_WAVE_TILING)
    torch.manual_seed(7)
    saved = (_lib.get_option(PF_OPT_GEMM_STAGED_RESID), _lib.get_option(PF_OPT_GEMM_WAVE_TILING))

    def run_all():
        outs = []
        for (B, S, K, N, r0) in [(2, 300, 384, 384, 40), (1, 3872, 1920, 1920, 0), (2, 777, 512, 1920, 5), (1, 128, 1920, 1920, 0)]:
            g = torch.Generator(device=DEV).manual_seed(B * 1000 + S)
            x = (torch.randn(B, S, K, device=DEV, generator=g) * 0.5).bfloat16()
            w = (torch.randn(N, K, device=DEV, generator=g) * 0.05).bfloat16()
            bias = torch.randn(N, device=DEV, generator=g) * 0.1
            resid = torch.randn(B, S, N, device=DEV, generator=g)
            gate = torch.randn(B, N, device=DEV, generator=g)
            ops.gemm(x, w, bias, PF_EPI_GATE_RESID, batches=B, rows_per_batch=S, row_begin=r0, row_count=S - r0, out=resid,
                     gate=gate, gate_batch_stride=N)
            y = torch.zeros(B, S, N, device=DEV, dtype=torch.bfloat16)
            ops.gemm(x, w, bias, PF_EPI_GELU_BF16, batches=B, rows_per_batch=S, row_begin=r0, row_count=S - r0, out=y)
            torch.cuda.synchronize()
            outs += [resid, y]
            if S == 300:     # and against fp32 math once
                want = F.gelu(x[:, r0:].float() @ w.float().t() + bias, approximate="tanh")
                assert _rel(y[:, r0:], want) < 8e-3
        return outs

    try:
        _lib.set_option(PF_OPT_GEMM_STAGED_RESID, 0)
        _lib.set_option(PF_OPT_GEMM_WAVE_TILING, 0)
        base = run_all()
        for staged, wave in ((1, 0), (0, 1), (1, 1)):
            _lib.set_option(PF_OPT_GEMM_STAGED_RESID, staged)
            _lib.set_option(PF_OPT_GEMM_WAVE_TILING, wave)
            got = run_all()
            for a, b in zip(base, got):
                assert torch.equal(a, b), (staged, wave)
    finally:
        _lib.set_option(PF_OPT_GEMM_STAGED_RESID, saved[0])
        _lib.set_option(PF_OPT_GEMM_WAVE_TILING, saved[1])
