"""The sequence-parallel peer stores on one GPU, bit for bit.

Under Ulysses sequence parallelism (sp.py, joint_step.StepLaunches) the exchange at the attention boundary has no copy
kernel: the QKV GEMM epilogue stores each head's rows into the owning rank's gathered q/k/v buffer (pf_gemm_desc.peer_*),
the attention epilogue stores each token chunk's output into its owner's `cat` buffer (pf_attn_desc.peer_*), and
pf_peer_bcast / pf_peer_barrier publish small results and order the remote stores.  A peer pointer is a global address, so
the same code runs when every "peer" buffer is an ordinary local allocation.  Here the ranks of one sp group are emulated
one after another in one process, each with an arena laid out like sp.PeerExchange's, and every descriptor comes from
sp.peer_store_args.  A GEMM row's bits do not depend on the launch's row range or on which GEMM kernel runs, and attention
heads are independent, so the emulated ranks must reproduce the single-GPU launches exactly (torch.equal).

Every arena byte the kernels must not write (guard bands around each region, the `cat` MLP columns) holds a NaN bit
pattern and is compared through an int16 view; the padded heads' q/k/v hold finite junk, as a re-sliced arena does."""
import ctypes as C

import pytest
import torch

from pyramid_flow_b200 import _lib, ops
from pyramid_flow_b200 import sp as SP
from pyramid_flow_b200._lib import PF_EPI_GATE_RESID, PF_EPI_GELU_BF16, PF_EPI_QKV_ROPE, PeerGroup
from pyramid_flow_b200.dit import build_seq_plan
from pyramid_flow_b200.joint_step import row_ranges

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN16 = 0x7FA5          # a quiet-NaN bf16 bit pattern
GUARD = 256             # bytes of NaN pattern before and after each arena region
SCALE = 0.125

# (text tokens, clip token grids (t, h, w)).  small: S = 77 + 523 = 600; at sp = 8 the chunks hold 75 rows, so the
# text / video boundary falls inside rank 1's chunk.  bench: the benchmarked step, S = 128 + 15360 = 15488; its chunks at
# sp = 4 / 8 (3872 / 1936 rows) are not multiples of 128, so q tiles straddle two ranks.
SEQS = {"small": (77, [(1, 5, 7), (2, 8, 13), (1, 14, 20)]),
        "bench": (128, [(28, 12, 20), (1, 24, 40), (1, 48, 80), (1, 48, 80)])}
# (heads, sp, sequence): 30 heads pad to 32 at sp 4 and 8 (the last rank owns 2 padded heads); 24 heads at sp 4 is the
# SD3 MMDiT layout
CASES = [(30, 2, "small"), (30, 4, "small"), (30, 8, "small"), (24, 4, "small"), (4, 2, "small"),
         (30, 4, "bench"), (30, 8, "bench")]
_PLANS = {}


def _plan(name):
    """The sequence plan of one CFG branch as the model builds it (padded text, several clips)."""
    if name not in _PLANS:
        text_len, grids = SEQS[name]
        mask = torch.ones(1, text_len, dtype=torch.int64)
        mask[0, text_len * 2 // 3:] = 0
        shapes = [(1, 16, t, 2 * h, 2 * w) for t, h, w in grids]
        _PLANS[name] = build_seq_plan(shapes, mask, (16, 24, 24), 2, DEV)
    return _PLANS[name]


def _i16(t):
    return t.contiguous().view(torch.int16) if t.dtype != torch.int16 else t


class _Arena:
    """One emulated rank's peer arena: qkv bf16 [3, Hg, S, 64] (its head group over the whole sequence) and cat bf16
    [S/sp, ldc] ([attention out | MLP hidden] of its token chunk), each with GUARD bytes before and after."""

    def __init__(self, seq, sl, hg, n_real, ldc, wa):
        a256 = lambda n: (n + 255) // 256 * 256
        self.hg, self.n_real, self.wa, self.ldc = hg, n_real, wa, ldc
        self.qkv_bytes, self.cat_bytes = 3 * hg * seq * 64 * 2, sl * ldc * 2
        self.off_qkv = GUARD
        self.off_cat = self.off_qkv + a256(self.qkv_bytes) + GUARD
        self.buf = torch.empty((self.off_cat + a256(self.cat_bytes) + GUARD) // 2, dtype=torch.int16, device=DEV)
        self.qkv = self.buf[self.off_qkv // 2:(self.off_qkv + self.qkv_bytes) // 2].view(torch.bfloat16).view(3, hg, seq, 64)
        self.cat = self.buf[self.off_cat // 2:(self.off_cat + self.cat_bytes) // 2].view(torch.bfloat16).view(sl, ldc)
        self.qkv_ptr = self.buf.data_ptr() + self.off_qkv
        self.cat_ptr = self.buf.data_ptr() + self.off_cat

    def fill(self, g):
        """NaN pattern everywhere, finite junk in the padded heads' q/k/v; returns the snapshot to compare against."""
        self.buf.fill_(NAN16)
        if self.n_real < self.hg:
            junk = torch.randn(3, self.hg - self.n_real, self.qkv.shape[2], 64, device=DEV, generator=g) * 100
            self.qkv[:, self.n_real:] = junk.bfloat16()
        self.snap = self.buf.clone()
        return self.snap

    def guards_intact(self):
        b, s = self.buf, self.snap
        q1, c1 = (self.off_qkv + self.qkv_bytes) // 2, (self.off_cat + self.cat_bytes) // 2
        return (torch.equal(b[:self.off_qkv // 2], s[:self.off_qkv // 2]) and torch.equal(b[q1:self.off_cat // 2], s[q1:self.off_cat // 2])
                and torch.equal(b[c1:], s[c1:]))

    def snap_view(self, region):
        s = self.snap
        if region == "qkv":
            return s[self.off_qkv // 2:(self.off_qkv + self.qkv_bytes) // 2].view(self.qkv.shape)
        return s[self.off_cat // 2:(self.off_cat + self.cat_bytes) // 2].view(self.cat.shape)


class _Group:
    """The emulated sp group of one (heads, sp, sequence) case."""

    def __init__(self, heads, sp, plan, mlp_cols):
        self.heads, self.sp, self.plan, self.seq = heads, sp, plan, plan.seq
        self.hp = SP.padded_heads(heads, sp)
        self.hg = self.hp // sp
        self.wa = self.hp * 64
        self.ldc = self.wa + mlp_cols
        self.bounds = [SP.chunk_bounds(self.seq, sp, r) for r in range(sp)]
        self.arenas = [_Arena(self.seq, c1 - c0, self.hg, max(0, min(self.hg, heads - r * self.hg)), self.ldc, self.wa)
                       for r, (c0, c1) in enumerate(self.bounds)]
        self.args = [SP.peer_store_args(self.seq, sp, r, self.hp, [a.qkv_ptr for a in self.arenas],
                                        [a.cat_ptr for a in self.arenas]) for r in range(sp)]

    def fill(self, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        for a in self.arenas:
            a.fill(g)

    def ranges(self, r):
        c0, c1 = self.bounds[r]
        return row_ranges(self.plan.text_len, self.seq, c0, c1)


def _qkv_weights(heads, g):
    d = heads * 64
    w = (torch.randn(3 * d, d, device=DEV, generator=g) * (0.7 / d ** 0.5)).bfloat16()
    b = torch.randn(3 * d, device=DEV, generator=g) * 0.1
    nq = 1 + 0.1 * torch.randn(64, device=DEV, generator=g)
    nk = 1 + 0.1 * torch.randn(64, device=DEV, generator=g)
    return w, b, nq, nk


def _qkv_single(xn, wts, heads, plan, rope, ranges, variants=(0, 0)):
    """The single-GPU QKV launches of StepLaunches.qkv over the whole sequence: q/k/v stacked [3, H, S, 64]."""
    s = plan.seq
    out = torch.zeros(3, heads, s, 64, device=DEV, dtype=torch.bfloat16)
    for j, (r0, rc) in enumerate(ranges):
        if rc == 0:
            continue
        w, b, nq, nk = wts[j]
        ops.gemm(xn, w, b, PF_EPI_QKV_ROPE, batches=1, rows_per_batch=s, row_begin=r0, row_count=rc, q_out=out[0][None],
                 k_out=out[1][None], v_out=out[2][None], rope=rope, q_norm_w=nq, k_norm_w=nk, norm_eps=1e-6, heads=heads,
                 head_dim=64, seq_len=s, kernel_variant=variants[j])
    return out


def _qkv_ranks(grp, xn, wts, rope, variants=(0, 0), dummy=None):
    """Every rank's QKV launches on its own chunk, storing into every rank's arena (StepLaunches.qkv with a parallel
    layout): the text and the video range as two launches, with their own weights."""
    for r, (c0, c1) in enumerate(grp.bounds):
        sl = c1 - c0
        xr = xn[:, c0:c1]
        for j, (r0, rc) in enumerate(grp.ranges(r)):
            if rc == 0:
                continue
            w, b, nq, nk = wts[j]
            ops.gemm(xr, w, b, PF_EPI_QKV_ROPE, batches=1, rows_per_batch=sl, row_begin=r0, row_count=rc, q_out=dummy,
                     k_out=dummy, v_out=dummy, rope=None if rope is None else rope[c0:c1], q_norm_w=nq, k_norm_w=nk,
                     norm_eps=1e-6, heads=grp.heads, head_dim=64, seq_len=sl, kernel_variant=variants[j], peer=grp.args[r][0])


def _attn_ranks(grp, q_row_begin=0):
    """Every rank's attention over its head group of the whole sequence, storing each token chunk into its owner's cat."""
    p = grp.plan
    for r, a in enumerate(grp.arenas):
        ops.attn_fwd(a.qkv[0][None], a.qkv[1][None], a.qkv[2][None], None, p.seg, p.time, p.sched, SCALE,
                     q_row_begin=q_row_begin, ldo=grp.ldc, peer=grp.args[r][1])


def _check_qkv(grp, ref):
    """Real heads equal the single-GPU q/k/v; padded-head junk, cat and guard bands are untouched."""
    for r, a in enumerate(grp.arenas):
        n = a.n_real
        assert torch.equal(a.qkv[:, :n], ref[:, r * grp.hg:r * grp.hg + n]), f"rank {r}: gathered q/k/v differ"
        assert torch.equal(_i16(a.qkv[:, n:]), a.snap_view("qkv")[:, n:]), f"rank {r}: padded heads written"
        assert torch.equal(_i16(a.cat), a.snap_view("cat")), f"rank {r}: cat written by the QKV epilogue"
        assert a.guards_intact(), f"rank {r}: guard band written"


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-20)).item()


def _qkv_ref_f32(xn, wts, heads, plan, rope, ranges):
    """fp32 restatement of the QKV_ROPE epilogue (test_kernels_gpu.py): bias, per-head RMSNorm of q and k, RoPE."""
    out = []
    for j, (r0, rc) in enumerate(ranges):
        w, b, nq, nk = wts[j]
        y = xn[0, r0:r0 + rc].float() @ w.float().t() + b
        parts = []
        for sec, t in enumerate(y.chunk(3, dim=-1)):
            t = t.view(rc, heads, 64)
            if sec < 2:
                t = t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + 1e-6) * (nq, nk)[sec]
                c, s_ = rope[r0:r0 + rc, :, 0][:, None, :], rope[r0:r0 + rc, :, 1][:, None, :]
                t2 = t.view(rc, heads, 32, 2)
                t = torch.stack([c * t2[..., 0] - s_ * t2[..., 1], s_ * t2[..., 0] + c * t2[..., 1]], -1).view(rc, heads, 64)
            parts.append(t.transpose(0, 1))
        out.append(torch.stack(parts))
    return torch.cat(out, dim=2)


@pytest.mark.parametrize("heads,sp,seq", CASES)
def test_qkv_scatter_matches_single_gpu(heads, sp, seq):
    plan = _plan(seq)
    grp = _Group(heads, sp, plan, 4 * heads * 64)
    g = torch.Generator(device=DEV).manual_seed(heads * 100 + sp)
    xn = (torch.randn(1, plan.seq, heads * 64, device=DEV, generator=g) * 0.5).bfloat16()
    wts = [_qkv_weights(heads, g), _qkv_weights(heads, g)]            # context (text rows) and video weights
    dummy = torch.full((64,), 3.0, device=DEV, dtype=torch.bfloat16)
    ranges = row_ranges(plan.text_len, plan.seq, 0, plan.seq)
    for rope in (plan.rope, None):
        ref = _qkv_single(xn, wts, heads, plan, rope, ranges)
        # the 256 x 128 cluster kernel and the 128 x 64 kernel on every range; the automatic choice (the 128 x 128 kernel on
        # the bench's 128-row text range) on the text rows
        for variants in ((1, 1), (2, 2), (0, 1)):
            grp.fill(variants[0] * 7 + variants[1])
            _qkv_ranks(grp, xn, wts, rope, variants, dummy)
            torch.cuda.synchronize()
            _check_qkv(grp, ref)
            assert bool((dummy == 3.0).all()), "q_out/k_out/v_out are ignored with peer stores"
        if seq == "small" and sp == 4 and rope is not None:
            # the emulated ranks are also right, not only consistent: the fp32 epilogue within test_kernels_gpu.py's bound
            want = _qkv_ref_f32(xn, wts, heads, plan, rope, ranges)
            got = torch.cat([a.qkv[:, :a.n_real] for a in grp.arenas], dim=1)
            assert _rel(got, want) < 8e-3


def _random_qkv(heads, s, g):
    return torch.stack([torch.randn(heads, s, 64, device=DEV, generator=g).bfloat16() for _ in range(3)])


def _fill_gathered(grp, qkv):
    """Put head group r of the single-GPU q/k/v into rank r's arena, as the QKV epilogues would have."""
    for r, a in enumerate(grp.arenas):
        a.qkv[:, :a.n_real] = qkv[:, r * grp.hg:r * grp.hg + a.n_real]
        a.snap = a.buf.clone()


@pytest.mark.parametrize("heads,sp,seq", CASES)
def test_attention_scatter_matches_single_gpu(heads, sp, seq):
    plan = _plan(seq)
    s = plan.seq
    grp = _Group(heads, sp, plan, 4 * heads * 64)
    g = torch.Generator(device=DEV).manual_seed(heads + sp)
    qkv = _random_qkv(heads, s, g)
    ref = torch.zeros(1, s, heads * 64, device=DEV, dtype=torch.bfloat16)
    ops.attn_fwd(qkv[0][None], qkv[1][None], qkv[2][None], ref, plan.seg, plan.time, plan.sched, SCALE)
    n_last = plan.last_tokens
    starts = [0] + ([((s - n_last) // 128) * 128] if seq == "small" else [])
    for qb in starts:
        grp.fill(qb + 1)
        _fill_gathered(grp, qkv)
        _attn_ranks(grp, q_row_begin=qb)
        torch.cuda.synchronize()
        for p, (a, (c0, c1)) in enumerate(zip(grp.arenas, grp.bounds)):
            lo = min(max(qb - c0, 0), c1 - c0)           # this chunk's rows below q_row_begin stay untouched
            assert torch.equal(a.cat[lo:, :heads * 64], ref[0, c0 + lo:c1]), f"rank {p}: attention rows differ"
            assert torch.equal(_i16(a.cat[:lo]), a.snap_view("cat")[:lo]), f"rank {p}: rows below q_row_begin written"
            assert bool(torch.isfinite(a.cat[lo:, heads * 64:grp.wa].float()).all()), f"rank {p}: padded heads not finite"
            assert torch.equal(_i16(a.cat[:, grp.wa:]), a.snap_view("cat")[:, grp.wa:]), f"rank {p}: MLP columns written"
            assert torch.equal(_i16(a.qkv), a.snap_view("qkv")), f"rank {p}: q/k/v written"
            assert a.guards_intact(), f"rank {p}: guard band written"


def _padk(w, heads, hp):
    """dit._pad_heads: zero input columns for the padded heads of a GEMM that reads the attention output."""
    d = heads * 64
    z = torch.zeros(w.shape[0], (hp - heads) * 64, device=w.device, dtype=w.dtype)
    return torch.cat([w[:, :d], z, w[:, d:]], dim=1).contiguous()


class _Block:
    """One joint (double) block's attention half and one single block, on one GPU and emulated over the sp ranks."""

    def __init__(self, heads, sp, plan, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        d = heads * 64
        self.heads, self.d, self.plan = heads, d, plan
        self.grp = _Group(heads, sp, plan, 4 * d)
        hp = self.grp.hp
        self.dbl_qkv = [_qkv_weights(heads, g), _qkv_weights(heads, g)]
        self.sgl_qkv = [_qkv_weights(heads, g)] * 2
        self.w_o = [(torch.randn(d, d, device=DEV, generator=g) * (0.7 / d ** 0.5)).bfloat16() for _ in range(2)]
        self.b_o = [torch.randn(d, device=DEV, generator=g) * 0.1 for _ in range(2)]
        self.w_mlp = (torch.randn(4 * d, d, device=DEV, generator=g) * (0.7 / d ** 0.5)).bfloat16()
        self.b_mlp = torch.randn(4 * d, device=DEV, generator=g) * 0.1
        self.w_out = (torch.randn(d, 5 * d, device=DEV, generator=g) * (0.7 / (5 * d) ** 0.5)).bfloat16()
        self.b_out = torch.randn(d, device=DEV, generator=g) * 0.1
        self.gate = torch.randn(1, 2 * d, device=DEV, generator=g)
        self.w_o_p = [_padk(w, heads, hp) for w in self.w_o]
        self.w_out_p = _padk(self.w_out, heads, hp)
        s = plan.seq
        # inputs: the LN-modulated rows of the two blocks and the fp32 residual stream
        self.xn = torch.empty(1, s, d, device=DEV, dtype=torch.bfloat16)
        self.xn2 = torch.empty_like(self.xn)
        self.h0 = torch.empty(1, s, d, device=DEV)
        self.hr = [torch.empty(1, c1 - c0, d, device=DEV) for c0, c1 in self.grp.bounds]
        self.dummy = torch.zeros(64, device=DEV, dtype=torch.bfloat16)
        self.new_inputs(seed + 1)

    def new_inputs(self, seed):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.xn.copy_((torch.randn(self.xn.shape, device=DEV, generator=g) * 0.5).bfloat16())
        self.xn2.copy_((torch.randn(self.xn.shape, device=DEV, generator=g) * 0.5).bfloat16())
        self.h0.copy_(torch.randn(self.h0.shape, device=DEV, generator=g))

    def single_gpu(self):
        """The block on one GPU (StepLaunches with no parallel layout): the residual stream after both blocks."""
        p, d, H, s = self.plan, self.d, self.heads, self.plan.seq
        wa, ldc = H * 64, H * 64 + 4 * d
        ranges = row_ranges(p.text_len, s, 0, s)
        h = self.h0.clone()
        cat = torch.zeros(1, s, ldc, device=DEV, dtype=torch.bfloat16)
        qkv = _qkv_single(self.xn, self.dbl_qkv, H, p, p.rope, ranges)
        ops.attn_fwd(qkv[0][None], qkv[1][None], qkv[2][None], cat, p.seg, p.time, p.sched, SCALE)
        for j, (r0, rc) in enumerate(ranges):
            ops.gemm(cat[:, :, :wa], self.w_o[j], self.b_o[j], PF_EPI_GATE_RESID, batches=1, rows_per_batch=s, row_begin=r0,
                     row_count=rc, out=h, ldo=d, gate=self.gate, gate_batch_stride=2 * d)
        qkv = _qkv_single(self.xn2, self.sgl_qkv, H, p, p.rope, ((0, s), (s, 0)))
        ops.gemm(self.xn2, self.w_mlp, self.b_mlp, PF_EPI_GELU_BF16, batches=1, rows_per_batch=s, row_begin=0, row_count=s,
                 out=cat, ldo=ldc, out_col_begin=wa)
        ops.attn_fwd(qkv[0][None], qkv[1][None], qkv[2][None], cat, p.seg, p.time, p.sched, SCALE)
        ops.gemm(cat, self.w_out, self.b_out, PF_EPI_GATE_RESID, batches=1, rows_per_batch=s, row_begin=0, row_count=s,
                 out=h, ldo=d, gate=self.gate[:, d:], gate_batch_stride=2 * d)
        return h

    def emulated(self):
        """The same block over the sp ranks, in rank order at every exchange: QKV of every rank, attention of every rank,
        then every rank's projections on its own `cat` with the head-padded weights; into self.hr (h0's rows first)."""
        grp, d, p = self.grp, self.d, self.plan
        for hr, (c0, c1) in zip(self.hr, grp.bounds):
            hr.copy_(self.h0[:, c0:c1])
        _qkv_ranks(grp, self.xn, self.dbl_qkv, p.rope, dummy=self.dummy)
        _attn_ranks(grp)
        for r, (a, hr) in enumerate(zip(grp.arenas, self.hr)):
            sl = hr.shape[1]
            for j, (r0, rc) in enumerate(grp.ranges(r)):
                if rc:
                    ops.gemm(a.cat[None, :, :grp.wa], self.w_o_p[j], self.b_o[j], PF_EPI_GATE_RESID, batches=1,
                             rows_per_batch=sl, row_begin=r0, row_count=rc, out=hr, ldo=d, gate=self.gate,
                             gate_batch_stride=2 * d)
        _qkv_ranks_single(grp, self.xn2, self.sgl_qkv, p.rope, self.dummy)
        for a, hr, (c0, c1) in zip(grp.arenas, self.hr, grp.bounds):
            ops.gemm(self.xn2[:, c0:c1], self.w_mlp, self.b_mlp, PF_EPI_GELU_BF16, batches=1, rows_per_batch=c1 - c0,
                     row_begin=0, row_count=c1 - c0, out=a.cat[None], ldo=grp.ldc, out_col_begin=grp.wa)
        _attn_ranks(grp)
        for a, hr in zip(grp.arenas, self.hr):
            sl = hr.shape[1]
            ops.gemm(a.cat[None], self.w_out_p, self.b_out, PF_EPI_GATE_RESID, batches=1, rows_per_batch=sl, row_begin=0,
                     row_count=sl, out=hr, ldo=d, gate=self.gate[:, d:], gate_batch_stride=2 * d)

    def check(self, ref):
        for r, (hr, (c0, c1)) in enumerate(zip(self.hr, self.grp.bounds)):
            # the padded heads' attention output is finite junk; their zero weight columns add exact zeros
            assert torch.equal(hr, ref[:, c0:c1]), f"rank {r}: residual rows differ (max |diff| " \
                f"{(hr - ref[:, c0:c1]).abs().max().item():.3e})"


def _qkv_ranks_single(grp, xn, wts, rope, dummy):
    """A single block's QKV: one launch over each rank's whole chunk."""
    for r, (c0, c1) in enumerate(grp.bounds):
        w, b, nq, nk = wts[0]
        ops.gemm(xn[:, c0:c1], w, b, PF_EPI_QKV_ROPE, batches=1, rows_per_batch=c1 - c0, row_begin=0, row_count=c1 - c0,
                 q_out=dummy, k_out=dummy, v_out=dummy, rope=rope[c0:c1], q_norm_w=nq, k_norm_w=nk, norm_eps=1e-6,
                 heads=grp.heads, head_dim=64, seq_len=c1 - c0, peer=grp.args[r][0])


@pytest.mark.parametrize("heads,sp,seq", [c for c in CASES if c[2] == "small"] + [(30, 8, "bench")])
def test_block_across_the_boundary_matches_single_gpu(heads, sp, seq):
    blk = _Block(heads, sp, _plan(seq), seed=heads * 10 + sp)
    ref = blk.single_gpu()
    blk.grp.fill(5)
    blk.emulated()
    torch.cuda.synchronize()
    blk.check(ref)
    for r, a in enumerate(blk.grp.arenas):
        assert a.guards_intact(), f"rank {r}: guard band written"


def test_block_across_the_boundary_under_graph_replay():
    """The bench replays the parallel step from a CUDA graph: the captured emulation, replayed on new inputs, gives the
    bits of an eager run on those inputs."""
    _lib.require_device()
    blk = _Block(30, 4, _plan("small"), seed=11)
    blk.grp.fill(5)
    blk.emulated()                                       # eager warm-up before capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        blk.emulated()
    blk.new_inputs(99)
    ref = blk.single_gpu()
    blk.grp.fill(6)
    blk.emulated()
    torch.cuda.synchronize()
    eager = [hr.clone() for hr in blk.hr]
    blk.check(ref)
    for seed in (99, 123):
        blk.new_inputs(seed)
        blk.grp.fill(6)
        for hr in blk.hr:
            hr.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        if seed == 99:
            for hr, e in zip(blk.hr, eager):
                assert torch.equal(hr, e)
        else:
            blk.check(blk.single_gpu())
        for r, a in enumerate(blk.grp.arenas):
            assert a.guards_intact(), f"rank {r}: guard band written"


# -- pf_peer_bcast ------------------------------------------------------------------------------------------------------
def _bcast(grp, src, nbytes, off):
    _lib.check(_lib.load().pf_peer_bcast(C.byref(grp), src, nbytes, off, _lib.stream_ptr()), "pf_peer_bcast")


# 16 B; 4112 B; 5 MB + 48 B, more than 296 blocks x 256 threads x 16 B, so the kernel's grid-stride loop runs
@pytest.mark.parametrize("nbytes", [16, 4112, 5 * 2 ** 20 + 48])
@pytest.mark.parametrize("n", [1, 2, 8])
def test_bcast_writes_every_member_and_nothing_else(n, nbytes):
    _lib.require_device()
    g = torch.Generator(device=DEV).manual_seed(n + nbytes)
    off = 16 * (n + 3)
    size = off + nbytes + 4096
    bufs = [torch.randint(0, 256, (size,), device=DEV, dtype=torch.uint8, generator=g) for _ in range(n)]
    before = [b.clone() for b in bufs]
    src = torch.randint(0, 256, (nbytes,), device=DEV, dtype=torch.uint8, generator=g)
    grp = PeerGroup()
    for i, b in enumerate(bufs):
        grp.ptr[i] = b.data_ptr()
    grp.n, grp.my_index = n, n - 1
    _bcast(grp, src.data_ptr(), nbytes, off)
    torch.cuda.synchronize()
    for i, (b, b0) in enumerate(zip(bufs, before)):
        assert torch.equal(b[off:off + nbytes], src), f"member {i}"
        assert torch.equal(b[:off], b0[:off]) and torch.equal(b[off + nbytes:], b0[off + nbytes:]), f"member {i}"


def test_bcast_from_the_local_slice():
    """StepLaunches.head(): src is the slice at the same offset of the local member's buffer (ptr[my_index])."""
    _lib.require_device()
    n, me, nbytes, off = 4, 2, 4112, 1040
    g = torch.Generator(device=DEV).manual_seed(3)
    bufs = [torch.randint(0, 256, (off + nbytes + 512,), device=DEV, dtype=torch.uint8, generator=g) for _ in range(n)]
    before = [b.clone() for b in bufs]
    grp = PeerGroup()
    for i, b in enumerate(bufs):
        grp.ptr[i] = b.data_ptr()
    grp.n, grp.my_index = n, me
    _bcast(grp, bufs[me].data_ptr() + off, nbytes, off)
    torch.cuda.synchronize()
    want = before[me][off:off + nbytes]
    for i, (b, b0) in enumerate(zip(bufs, before)):
        assert torch.equal(b[off:off + nbytes], want), f"member {i}"
        assert torch.equal(b[:off], b0[:off]) and torch.equal(b[off + nbytes:], b0[off + nbytes:]), f"member {i}"


# -- pf_peer_barrier ----------------------------------------------------------------------------------------------------
def _u32(x):
    return int(x) & 0xFFFFFFFF


def _i32(x):
    x = _u32(x)
    return x - (1 << 32) if x & 0x80000000 else x


class _Barrier:
    """n members' flag arrays (PF_MAX_PEERS uint32 each, separate allocations) and this member's epoch counter."""

    def __init__(self, n, me, epoch):
        self.n, self.me = n, me
        self.flags = [torch.full((8,), 0x5A5A5A5A, device=DEV, dtype=torch.int32) for _ in range(n)]
        self.epoch = torch.tensor([_i32(epoch)], device=DEV, dtype=torch.int32)
        self.grp = PeerGroup()
        for i, f in enumerate(self.flags):
            self.grp.ptr[i] = f.data_ptr()
        self.grp.n, self.grp.my_index = n, me

    def next_epoch(self):
        return _u32(self.epoch.item() + 1)

    def arrive_others(self, e):
        """What the other members' barrier kernels would have published: their slot in my flag array reaches e."""
        for i in range(self.n):
            if i != self.me:
                self.flags[self.me][i] = _i32(e)
        torch.cuda.synchronize()

    def assert_no_wait(self):
        """No launch may wait on a flag that nobody writes: every slot the kernel polls already holds v, int32(v - e) >= 0."""
        e = self.next_epoch()
        mine = self.flags[self.me].cpu()
        for i in range(self.n):
            if i != self.me:
                assert _i32(_u32(mine[i].item()) - e) >= 0, f"slot {i} would be polled without an arrival"

    def launch(self, check=True):
        if check:                      # (not while capturing: the host read would break the capture)
            self.assert_no_wait()
        _lib.check(_lib.load().pf_peer_barrier(C.byref(self.grp), self.epoch.data_ptr(), _lib.stream_ptr()),
                   "pf_peer_barrier")


def test_barrier_single_member_advances_per_launch_and_per_replay():
    _lib.require_device()
    bar = _Barrier(1, 0, 41)
    for e in (42, 43):
        bar.launch()
        torch.cuda.synchronize()
        assert _u32(bar.epoch.item()) == e and _u32(bar.flags[0][0].item()) == e
        assert bool((bar.flags[0][1:] == 0x5A5A5A5A).all())
    graph = torch.cuda.CUDAGraph()
    bar.assert_no_wait()
    with torch.cuda.graph(graph):
        bar.launch(check=False)
    for e in (44, 45, 46):   # capture does not run the kernel
        assert bar.next_epoch() == e
        bar.assert_no_wait()
        graph.replay()
        torch.cuda.synchronize()
        assert _u32(bar.epoch.item()) == e and _u32(bar.flags[0][0].item()) == e


def test_barrier_publishes_my_slot_in_every_member():
    """n = 4, my_index = 2: epoch e goes into slot 2 of every member's flag array, nothing else changes; the counter wraps
    through 2^32 with the signed comparison of the wait."""
    _lib.require_device()
    n, me = 4, 2
    bar = _Barrier(n, me, 0xFFFFFFFD)
    for e in (0xFFFFFFFE, 0xFFFFFFFF, 0, 1):
        assert bar.next_epoch() == e
        bar.arrive_others(e if e != 0xFFFFFFFF else _u32(e + 3))      # one round with the others already ahead
        before = [f.clone() for f in bar.flags]
        bar.launch()
        torch.cuda.synchronize()
        assert _u32(bar.epoch.item()) == e
        for i, (f, f0) in enumerate(zip(bar.flags, before)):
            want = f0.clone()
            want[me] = _i32(e)
            assert torch.equal(f, want), f"member {i}: {f.tolist()} != {want.tolist()}"
