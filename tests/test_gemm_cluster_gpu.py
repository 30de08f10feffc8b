"""The 256 x 128 two-CTA cluster GEMM kernel through pf_gemm_bf16, against fp32 PyTorch with the tolerances of
test_kernels_gpu.py: every epilogue at the DiT step's shapes and at the tile-edge cases (odd m-tile count, ragged row ranges
with offsets, ragged last pair of a batch, fewer tiles than SMs, K not a multiple of 64), plus the bitwise claims (a tile's
rows do not depend on the launch they are computed in, nor on which of the three GEMM kernels runs)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
H_STEP, HD = 30, 64


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-20)).item()


def _f32_tol(K):
    # test_kernels_gpu.py's 1e-5 for fp32 outputs, widened like the fp32 accumulation error (sqrt K) past K = 1920
    return 1e-5 * max(1.0, (K / 1920) ** 0.5)


def _inputs(B, S, K, N, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn(B, S, K, device=DEV, generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) * (0.7 / K ** 0.5)).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g) * 0.1
    return g, x, w, bias


def _run(epi, B, S, K, N, r0, rc, *, heads=0, out_pad=0, out_shift=0, variant=1, seed=0):
    """One launch of `epi` over rows [r0, r0 + rc) of each batch; returns (outputs, fp32 references, untouched-row check)."""
    from pyramid_flow_b200 import ops
    from pyramid_flow_b200._lib import PF_EPI_GATE_RESID, PF_EPI_GELU_BF16, PF_EPI_QKV_ROPE, PF_EPI_STORE_BF16
    g, x, w, bias = _inputs(B, S, K, N, seed)
    y = x[:, r0:r0 + rc].float() @ w.float().t() + bias
    if epi == PF_EPI_QKV_ROPE:
        H = heads
        qn = 1 + 0.1 * torch.randn(HD, device=DEV, generator=g)
        kn = 1 + 0.1 * torch.randn(HD, device=DEV, generator=g)
        ang = torch.randn(S, HD // 2, device=DEV, generator=g)
        rope = torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous()
        q, k, v = (torch.zeros(B, H, S, HD, device=DEV, dtype=torch.bfloat16) for _ in range(3))
        ops.gemm(x, w, bias, epi, batches=B, rows_per_batch=S, row_begin=r0, row_count=rc, q_out=q, k_out=k, v_out=v,
                 rope=rope, q_norm_w=qn, k_norm_w=kn, heads=H, head_dim=HD, seq_len=S, kernel_variant=variant)
        yq, yk, yv = y.chunk(3, dim=-1)

        def nr(t, wn):
            t = t.view(B, rc, H, HD)
            t = t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6) * wn
            c, s_ = rope[r0:r0 + rc, :, 0][None, :, None, :], rope[r0:r0 + rc, :, 1][None, :, None, :]
            t2 = t.view(B, rc, H, HD // 2, 2)
            return torch.stack([c * t2[..., 0] - s_ * t2[..., 1], s_ * t2[..., 0] + c * t2[..., 1]], -1).view(B, rc, H, HD).transpose(1, 2)
        outs = [q[:, :, r0:r0 + rc], k[:, :, r0:r0 + rc], v[:, :, r0:r0 + rc]]
        refs = [nr(yq, qn), nr(yk, kn), yv.reshape(B, rc, H, HD).transpose(1, 2)]
        untouched = bool((q[:, :, :r0] == 0).all() and (q[:, :, r0 + rc:] == 0).all())
        return outs, refs, untouched, 8e-3
    ob = S + out_pad
    orb = r0 + out_shift
    if epi == PF_EPI_GATE_RESID:
        resid = torch.randn(B, ob, N, device=DEV, generator=g)
        r_in = resid.clone()
        gate = torch.randn(B, 2 * N, device=DEV, generator=g)
        ops.gemm(x, w, bias, epi, batches=B, rows_per_batch=S, row_begin=r0, row_count=rc, out=resid, ldo=N,
                 out_batch_rows=ob, out_row_begin=orb, gate=gate[:, N:], gate_batch_stride=2 * N, kernel_variant=variant)
        ref = r_in[:, orb:orb + rc] + gate[:, None, N:] * y
        untouched = bool(torch.equal(resid[:, :orb], r_in[:, :orb]) and torch.equal(resid[:, orb + rc:], r_in[:, orb + rc:]))
        return [resid[:, orb:orb + rc]], [ref], untouched, _f32_tol(K)
    f32 = epi not in (PF_EPI_GELU_BF16, PF_EPI_STORE_BF16)
    out = torch.zeros(B, ob, N, device=DEV, dtype=torch.float32 if f32 else torch.bfloat16)
    ops.gemm(x, w, bias, epi, batches=B, rows_per_batch=S, row_begin=r0, row_count=rc, out=out, out_batch_rows=ob,
             out_row_begin=orb, kernel_variant=variant)
    ref = F.gelu(y, approximate="tanh") if epi == PF_EPI_GELU_BF16 else y
    untouched = bool((out[:, :orb] == 0).all() and (out[:, orb + rc:] == 0).all())
    return [out[:, orb:orb + rc]], [ref], untouched, (_f32_tol(K) if f32 else 8e-3)


def _check(res):
    outs, refs, untouched, tol = res
    torch.cuda.synchronize()
    for o, r in zip(outs, refs):
        assert _rel(o, r) < tol
    assert untouched


# the step's GEMM families (B=2, S=15488 = 128 text + 15360 video tokens, 30 heads): (epilogue name, r0, rows, N, K)
STEP = [("QKV_ROPE", 128, 15360, 3 * 1920, 1920), ("QKV_ROPE", 0, 128, 3 * 1920, 1920), ("QKV_ROPE", 0, 15488, 3 * 1920, 1920),
        ("GELU_BF16", 128, 15360, 4 * 1920, 1920), ("GELU_BF16", 0, 15488, 4 * 1920, 1920),
        ("GATE_RESID", 128, 15360, 1920, 1920), ("GATE_RESID", 128, 15360, 1920, 4 * 1920),
        ("GATE_RESID", 0, 15488, 1920, 5 * 1920), ("GATE_RESID", 0, 128, 1920, 4 * 1920)]


@pytest.mark.parametrize("name,r0,rc,n,k", STEP)
def test_gemm_step_shapes(name, r0, rc, n, k):
    from pyramid_flow_b200 import _lib
    epi = getattr(_lib, "PF_EPI_" + name)
    _check(_run(epi, 2, 15488, k, n, r0, rc, heads=H_STEP, variant=0))


EPIS = ["STORE_BF16", "GELU_BF16", "STORE_F32", "GATE_RESID", "QKV_ROPE"]
# (B, S, K, N, r0, rc, out_pad, out_shift): odd m-tile count (3 tiles: the last pair's partner has no rows); ragged range
# with row / output offsets; batches=2 with a ragged last pair; fewer tiles than SMs; K not a multiple of 64
EDGES = [(1, 768, 256, 384, 0, 600, 0, 0), (1, 1000, 320, 384, 37, 700, 50, 11), (2, 900, 192, 768, 3, 890, 0, 0),
         (1, 128, 128, 384, 0, 128, 0, 0), (2, 520, 1000, 384, 8, 500, 16, 4)]


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("name", EPIS)
def test_gemm_cluster_edges(name, edge):
    from pyramid_flow_b200 import _lib
    B, S, K, N, r0, rc, pad, shift = edge
    epi = getattr(_lib, "PF_EPI_" + name)
    if epi == _lib.PF_EPI_QKV_ROPE:
        if pad or shift:
            pytest.skip("QKV positions are out_row_begin + m (no separate output rows)")
        _check(_run(epi, B, S, K, N, r0, rc, heads=N // (3 * HD)))
    else:
        _check(_run(epi, B, S, K, N, r0, rc, out_pad=pad, out_shift=shift))


@pytest.mark.parametrize("name", EPIS)
def test_gemm_cluster_bits_match_other_kernels_and_launches(name):
    """Same bits from the cluster kernel (variant 1), the 128 x 64 kernel (variant 2), and a separate launch of one
    256-row tile's rows."""
    from pyramid_flow_b200 import _lib
    epi = getattr(_lib, "PF_EPI_" + name)
    B, S, K, N = 2, 1024, 448, 384
    kw = dict(heads=N // (3 * HD)) if epi == _lib.PF_EPI_QKV_ROPE else {}
    whole = _run(epi, B, S, K, N, 0, S, variant=1, **kw)[0]
    other = _run(epi, B, S, K, N, 0, S, variant=2, **kw)[0]
    part = _run(epi, B, S, K, N, 256, 256, variant=1, **kw)[0]
    torch.cuda.synchronize()
    for a, b, c in zip(whole, other, part):
        assert torch.equal(a, b)
        assert torch.equal(a[:, :, 256:512] if epi == _lib.PF_EPI_QKV_ROPE else a[:, 256:512], c)


@pytest.mark.parametrize("edge", [EDGES[1], EDGES[2]])
def test_gemm_cluster_qkv_gelu_matches_split_launches(edge):
    """The fused q|k|v|mlp epilogue gives the bits of QKV_ROPE on the first 3*H*64 columns and GELU_BF16 on the rest."""
    from pyramid_flow_b200 import ops
    from pyramid_flow_b200._lib import PF_EPI_GELU_BF16, PF_EPI_QKV_GELU, PF_EPI_QKV_ROPE
    B, S, K, _, r0, rc, _, _ = edge
    H, nm = 2, 512
    nq = 3 * H * HD
    g, x, w, bias = _inputs(B, S, K, nq + nm, 5)
    qn, kn = 1 + 0.1 * torch.randn(HD, device=DEV, generator=g), 1 + 0.1 * torch.randn(HD, device=DEV, generator=g)
    ang = torch.randn(S, HD // 2, device=DEV, generator=g)
    rope = torch.stack([ang.cos(), ang.sin()], dim=-1).contiguous()
    qkv = dict(rope=rope, q_norm_w=qn, k_norm_w=kn, heads=H, head_dim=HD, seq_len=S)
    fused = [torch.zeros(B, H, S, HD, device=DEV, dtype=torch.bfloat16) for _ in range(3)]
    split = [torch.zeros_like(fused[0]) for _ in range(3)]
    cat_f = torch.zeros(B, S, nm + 64, device=DEV, dtype=torch.bfloat16)
    cat_s = torch.zeros_like(cat_f)
    ops.gemm(x, w, bias, PF_EPI_QKV_GELU, batches=B, rows_per_batch=S, row_begin=r0, row_count=rc, out=cat_f,
             out_col_begin=64, q_out=fused[0], k_out=fused[1], v_out=fused[2], n_split=nq, kernel_variant=1, **qkv)
    ops.gemm(x, w[:nq].contiguous(), bias[:nq].contiguous(), PF_EPI_QKV_ROPE, batches=B, rows_per_batch=S, row_begin=r0,
             row_count=rc, q_out=split[0], k_out=split[1], v_out=split[2], kernel_variant=1, **qkv)
    ops.gemm(x, w[nq:].contiguous(), bias[nq:].contiguous(), PF_EPI_GELU_BF16, batches=B, rows_per_batch=S, row_begin=r0,
             row_count=rc, out=cat_s, out_col_begin=64, kernel_variant=1)
    torch.cuda.synchronize()
    for a, b in zip(fused, split):
        assert torch.equal(a, b)
    assert torch.equal(cat_f, cat_s)
    want = F.gelu(x[:, r0:r0 + rc].float() @ w[nq:].float().t() + bias[nq:], approximate="tanh")
    assert _rel(cat_f[:, r0:r0 + rc, 64:], want) < 8e-3
