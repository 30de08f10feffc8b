"""Exact mask coverage of the attention kernels on the H100, by identity-V probes (tests/attn_probe.py): the kernels print
their probability matrix (forward, dV) or their dS matrix (dQ, dK), and every element is compared with an fp64 attention of
the same bf16 inputs.  A masked pair must be exactly 0, an allowed one non-zero and within a bound derived from the
kernels' arithmetic, so a column mis-masked at a tile edge, a partial tile treated as full, a skipped kv tile or a leak from
a tail row or column fails here.  The sensitivity tests feed the kernels a deliberately wrong (in-bounds) schedule and
require that the probes report exactly the planted block."""
import ctypes as C
from dataclasses import dataclass

import pytest
import torch

from oracle import flux_oracle as FO
from pyramid_flow_b200 import _lib, ops
from pyramid_flow_b200._lib import AttnTextDesc
from pyramid_flow_b200.dit import build_seq_plan
from tests import attn_probe as AP

pytestmark = pytest.mark.gpu
DEV = "cuda"
SCALE = AP.SCALE

# the pyramid of test_plan_cpu.py: two history frames, one mid-resolution frame, the current frame (S = 1448)
PYRAMID_SHAPES = [(2, 16, 2, 12, 20), (2, 16, 1, 24, 40), (2, 16, 1, 48, 80)]
# the benchmarked step (bench.py step_clip_shapes: miniFLUX 768p, unit 30, stage 2; S = 15488)
STEP_SHAPES = [(2, 16, 28, 24, 40), (2, 16, 1, 48, 80), (2, 16, 1, 96, 160), (2, 16, 1, 96, 160)]


@dataclass
class Layout:
    seg: torch.Tensor         # device int32 [B, S]
    time: torch.Tensor
    sched: torch.Tensor       # device int32 [B, q_tiles, stride]
    psched: object            # ops.PairSchedule on the device (variants 0x10 / 0x20)
    allowed: torch.Tensor     # device bool [B, S, S]
    distinct: bool            # per-head q and k (False: one q and k copied to every head)


def _plan_layout(shapes, mask, distinct=True) -> Layout:
    plan = build_seq_plan(shapes, mask, (16, 24, 24), 2, DEV)
    # the reference's dense mask (F:341-349) on the oracle's ids, not a restatement of the plan's
    seg_o = FO.token_segments(mask, plan.video_len).to(DEV)
    allowed = FO.attention_mask(seg_o, FO.sequence_ids(shapes, mask.shape[1])[:, 0].to(DEV))[:, 0]
    return Layout(plan.seg, plan.time, plan.sched, plan.sched2, allowed, distinct)


def _ids_layout(seg, time) -> Layout:
    sched, _ = ops.attn_build_schedule(seg, time)
    psched = ops.attn_build_pair_schedule(sched, seg.shape[1], seg, time).to(DEV)
    seg, time = seg.to(DEV), time.to(DEV)
    return Layout(seg, time, sched.to(DEV), psched, AP.dense_mask(seg, time), True)


def _fwd_layout(name) -> Layout:
    if name == "text77":            # text tokens only: one partial tile
        return _ids_layout(torch.ones(1, 77, dtype=torch.int32), torch.zeros(1, 77, dtype=torch.int32))
    if name == "joint1000":         # the SD3 joint sequence: one segment, one time, a tail tile
        return _ids_layout(torch.ones(1, 1000, dtype=torch.int32), torch.zeros(1, 1000, dtype=torch.int32))
    if name == "pyramid":           # history clips, text padded in sample 0 only
        mask = torch.ones(2, 128, dtype=torch.long)
        mask[0, 37:] = 0
        return _plan_layout(PYRAMID_SHAPES, mask)
    if name == "frames40":          # 40-token frames: every q tile meets only partial kv tiles
        return _ids_layout(*AP.restated_layout(2, 24, [(6, 40)]))
    if name == "random_ids":        # seg / time drawn per token: every tile partial, masks with holes
        return _ids_layout(*AP.random_ids_layout(2, 677, torch.Generator().manual_seed(5)))
    if name == "step15488":         # the benchmarked step, different text padding per sample
        mask = torch.ones(2, 128, dtype=torch.long)
        mask[0, 77:] = 0
        mask[1, 23:] = 0
        return _plan_layout(STEP_SHAPES, mask, distinct=False)
    raise KeyError(name)


def _fwd(q, k, v, lay: Layout, sched=None, **kw) -> torch.Tensor:
    """The probe launch: out [B, S, H * 64] is a view of a sentinel-filled buffer 64 columns wider, which must stay untouched."""
    b, h, s, _ = q.shape
    buf = torch.full((b, s, h * 64 + 64), AP.SENTINEL, device=DEV, dtype=torch.bfloat16)
    ops.attn_fwd(q, k, v, buf[..., :h * 64], lay.seg, lay.time, lay.sched if sched is None else sched, SCALE,
                 pair_sched=lay.psched, **kw)
    torch.cuda.synchronize()
    assert bool((buf[..., h * 64:] == AP.SENTINEL).all()), "write past the output columns"
    return buf[..., :h * 64]


def _fwd_probe(lay: Layout, seed: int):
    b, s = lay.seg.shape
    h = AP.heads_for(s)
    g = torch.Generator().manual_seed(seed)
    q, k = (AP.random_heads(b, s, h, g, DEV, lay.distinct) for _ in range(2))
    return q, k, AP.identity_heads(b, s, h, DEV)


def _fwd_reports(out, q, k, lay: Layout, name: str):
    bound = AP.rel_bound_fwd(SCALE, AP.norm_product_max(q, k))
    for bi in range(out.shape[0]):      # one sample at a time: the fp64 matrices of the step are 1.9 GB each
        p_ref, lse_ref = AP.fwd_reference(q[bi:bi + 1], k[bi:bi + 1], lay.allowed[bi:bi + 1], SCALE, lay.distinct)
        yield AP.check_probs(f"{name} forward, sample {bi}", out[bi:bi + 1], p_ref, lay.allowed[bi:bi + 1], bound), lse_ref
        del p_ref


@pytest.mark.parametrize("name", ["text77", "joint1000", "pyramid", "frames40", "random_ids", "step15488"])
def test_forward_probe(name):
    _lib.require_device()
    lay = _fwd_layout(name)
    q, k, v = _fwd_probe(lay, seed=len(name))
    b, h, s, _ = q.shape
    lse = torch.full((b, h, s), float("nan"), device=DEV)
    out = _fwd(q, k, v, lay, lse=lse)
    # lse: fp32 of the scores' error (scale EPS_ACC |q| |k|) plus fp32 rounding of a magnitude below 32
    lse_tol = SCALE * AP.EPS_ACC * AP.norm_product_max(q, k) + 2.0 ** -18 * 32
    worst, lse_err = 0.0, 0.0
    for bi, (rep, lse_ref) in enumerate(_fwd_reports(out, q, k, lay, name)):
        assert rep.ok(), str(rep)
        worst = max(worst, rep.worst)
        lse_err = max(lse_err, (lse[bi:bi + 1].double() - lse_ref).abs().max().item())
    print(f"{name}: S={s}, H={h}: worst relative error of P {worst:.3e} (bound {rep.rel_bound:.3e}); "
          f"lse max abs error {lse_err:.2e} (bound {lse_tol:.2e})")
    assert lse_err <= lse_tol

    # every accepted variant, and a second run, give the same bits; lse is repeatable too
    for variant in (3, 0x10, 0x20, 0):
        assert torch.equal(_fwd(q, k, v, lay, variant=variant), out), variant
    lse2 = torch.full_like(lse, float("nan"))
    _fwd(q, k, v, lay, lse=lse2)
    assert torch.equal(lse, lse2)
    # q_row_begin: rows at and after it keep their bits, rows before it keep the sentinel
    for qb in sorted({((s - 1) // 128) * 128, (s // 256) * 128} - {0}):
        o2 = _fwd(q, k, v, lay, q_row_begin=qb)
        assert torch.equal(o2[:, qb:], out[:, qb:]) and bool((o2[:, :qb] == AP.SENTINEL).all()), qb


# ---- backward ----------------------------------------------------------------------------------------------------------
# the layouts of test_train_attn_gpu.py (B = 2, text padded differently per sample) plus random ids
BWD_CASES = {
    "pyramid": (128, [(2, 48), (1, 96), (1, 384)], True),
    "all_partial": (24, [(6, 40)], True),
    "no_causal": (77, [(1, 60), (2, 150)], False),
}


def _bwd_layout(case):
    if case == "random_ids":
        return AP.random_ids_layout(2, 405, torch.Generator().manual_seed(9))
    return AP.restated_layout(2, *BWD_CASES[case])


def _bwd_probe(case, probe, sched=None, kv_sched=None, runs=1):
    """Run the forward (correct schedule) and the backward (the given schedules) on the probe's inputs.
    -> (report of the probed gradient, [(dq, dk, dv) per run])."""
    seg, time = _bwd_layout(case)
    b, s = seg.shape
    h = AP.heads_for(s)
    g = torch.Generator().manual_seed(len(case) * 3 + ["dv", "dq", "dk"].index(probe))
    ident = lambda: AP.identity_heads(b, s, h, DEV)
    rnd = lambda: AP.random_heads(b, s, h, g, DEV)
    q = ident() if probe == "dk" else rnd()
    k = ident() if probe == "dq" else rnd()
    v = rnd()
    dout = AP.head_columns(ident() if probe == "dv" else rnd()).contiguous()
    tile_sched, _ = ops.attn_build_schedule(seg, time)
    kv = ops.attn_build_kv_schedule(tile_sched, s)
    segd, timed = seg.to(DEV), time.to(DEV)
    out = torch.zeros(b, s, h * 64, device=DEV, dtype=torch.bfloat16)
    lse = torch.zeros(b, h, s, device=DEV)
    ops.attn_fwd(q, k, v, out, segd, timed, tile_sched.to(DEV), SCALE, lse=lse)
    sched_d = (tile_sched if sched is None else sched).to(DEV)
    kv_d = (kv if kv_sched is None else kv_sched).to(DEV)
    grads = []
    for _ in range(runs):
        dq, dk, dv = (torch.full_like(q, AP.SENTINEL) for _ in range(3))
        ops.attn_bwd(q, k, v, out, dout, lse, segd, timed, sched_d, kv_d, SCALE, dq, dk, dv)
        torch.cuda.synchronize()
        grads.append((dq, dk, dv))
    dq, dk, dv = grads[0]
    allowed = AP.dense_mask(segd, timed)
    ref = AP.bwd_reference(q, k, v, out, dout, allowed, SCALE)
    if probe == "dv":       # dV[b, h, kv, d] = P_h[64 h + d, kv]
        rep = AP.check_probs(f"{case} dV", AP.head_columns(dv), ref.pt, allowed.transpose(1, 2), ref.rel_dv)
    elif probe == "dq":     # dQ[b, h, q, d] = scale dS_h[q, 64 h + d]
        rep = AP.check_grads(f"{case} dQ", AP.head_columns(dq) / SCALE, ref.ds, ref.ds_bound, allowed)
    else:                   # dK[b, h, kv, d] = scale dS_h[64 h + d, kv]
        rep = AP.check_grads(f"{case} dK", AP.head_columns(dk) / SCALE, ref.dst, ref.dst_bound, allowed.transpose(1, 2))
    return rep, grads, (tile_sched, kv)


@pytest.mark.parametrize("probe", ["dv", "dq", "dk"])
@pytest.mark.parametrize("case", list(BWD_CASES) + ["random_ids"])
def test_backward_probe(case, probe):
    _lib.require_device()
    rep, grads, _ = _bwd_probe(case, probe, runs=2)
    print(str(rep).splitlines()[0])
    assert rep.ok(), str(rep)
    for a, b in zip(*grads):
        assert torch.equal(a, b), f"{case} {probe}: two runs differ"


# ---- sensitivity: a planted schedule fault is reported exactly where it was planted -----------------------------------
def _entry_index(sched, b, row, tile):
    ents = sched[b, row, 1:1 + int(sched[b, row, 0])].tolist()
    return [e >> 1 for e in ents].index(tile)


def _assert_fault_confined(rep: AP.Report, block: torch.Tensor, rows: torch.Tensor):
    block, rows = block.to(rep.leaked.device), rows.to(rep.leaked.device)
    print(str(rep))
    assert not rep.ok(), "the probe missed the planted fault"
    assert not bool((rep.exact_violations() & ~block).any()), "exact-rule violations outside the planted block"
    assert not bool((rep.inexact & ~rows).any()), "mismatches outside the planted block's rows"


def test_forward_probe_sees_a_dropped_kv_tile():
    lay = _fwd_layout("pyramid")
    sched = lay.sched.cpu()
    b, qt, kt = 1, 9, 3                 # a current-frame q tile of sample 1 and a fully allowed history kv tile
    i = _entry_index(sched, b, qt, kt)
    assert int(sched[b, qt, 1 + i]) & 1 == 0
    q, k, v = _fwd_probe(lay, seed=1)
    out = _fwd(q, k, v, lay, sched=AP.drop_entry(sched, b, qt, i).to(DEV))
    for rep, _ in _fwd_reports(out, q, k, lay, "dropped kv tile"):
        if rep.name.endswith(f"sample {b}"):
            shape = (1, *out.shape[1:])
            block = AP.tile_region(shape, 0, qt, kt)
            _assert_fault_confined(rep, block, AP.tile_region(shape, 0, qt))
            assert torch.equal(rep.missing, block.to(DEV) & AP.pad_cols(lay.allowed[b:b + 1], out.shape[-1], False))
        else:
            assert rep.ok(), str(rep)


def test_forward_probe_sees_a_partial_tile_run_as_full():
    lay = _fwd_layout("pyramid")
    sched = lay.sched.cpu()
    b, qt, kt = 0, 9, 0                 # sample 0's text tile holds padded keys (seg 0): partial, and not the tail tile
    i = _entry_index(sched, b, qt, kt)
    assert int(sched[b, qt, 1 + i]) & 1 == 1 and kt < sched.shape[1] - 1
    q, k, v = _fwd_probe(lay, seed=2)
    out = _fwd(q, k, v, lay, sched=AP.clear_partial(sched, b, qt, i).to(DEV))
    for rep, _ in _fwd_reports(out, q, k, lay, "partial tile run as full"):
        if rep.name.endswith(f"sample {b}"):
            shape = (1, *out.shape[1:])
            block = AP.tile_region(shape, 0, qt, kt)
            _assert_fault_confined(rep, block, AP.tile_region(shape, 0, qt))
            assert torch.equal(rep.leaked, block.to(DEV) & ~AP.pad_cols(lay.allowed[b:b + 1], out.shape[-1], False))
        else:
            assert rep.ok(), str(rep)


@pytest.mark.parametrize("probe", ["dv", "dk"])
def test_backward_probes_see_a_dropped_kv_schedule_entry(probe):
    _, _, (_, kv) = _bwd_probe("pyramid", probe)
    b, kt, qt = 1, 2, 5                 # kv tile 2 (history frames) of sample 1, seen by the last (tail) q tile
    mutated = AP.drop_entry(kv, b, kt, _entry_index(kv, b, kt, qt))
    rep, _, _ = _bwd_probe("pyramid", probe, kv_sched=mutated)
    shape = rep.leaked.shape            # [B, kv, q]
    block = AP.tile_region(shape, b, kt, qt)
    _assert_fault_confined(rep, block, block)
    assert bool(rep.missing.any())


def test_backward_dq_probe_sees_a_dropped_tile_schedule_entry():
    _, _, (tile_sched, _) = _bwd_probe("pyramid", "dq")
    b, qt, kt = 1, 5, 2
    rep, _, _ = _bwd_probe("pyramid", "dq", sched=AP.drop_entry(tile_sched, b, qt, _entry_index(tile_sched, b, qt, kt)))
    block = AP.tile_region(rep.leaked.shape, b, qt, kt)      # [B, q, kv]
    _assert_fault_confined(rep, block, block)
    assert bool(rep.missing.any())


# ---- text attention ----------------------------------------------------------------------------------------------------
def _text_case(seq, heads, batch, key_mask, causal, g):
    q, k = (AP.random_heads(batch, seq, heads, g, DEV) for _ in range(2))
    v = AP.identity_heads(batch, seq, heads, DEV)
    qkv = torch.cat([AP.head_columns(t) for t in (q, k, v)], -1).reshape(batch * seq, 3 * heads * 64).contiguous()
    allowed = key_mask.bool()[:, None, :].expand(batch, seq, seq)
    if causal:
        allowed = allowed & torch.ones(seq, seq, dtype=torch.bool, device=DEV).tril()
    return q, k, qkv, allowed


@pytest.mark.parametrize("seq", [1, 7, 77, 128, 200, 256])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("with_bias", [False, True])
def test_text_probe(seq, causal, with_bias):
    _lib.require_device()
    heads = AP.heads_for(seq) + 1       # one head more than the probe needs: its columns lie past seq and must be 0
    g = torch.Generator().manual_seed(seq * 4 + 2 * causal + with_bias)
    key_mask = torch.ones(3, seq, dtype=torch.int32, device=DEV)
    key_mask[0, 1:] = 0                 # a valid prefix of length 1
    key_mask[2, seq // 4:seq // 2] = 0  # holes in the middle (the mask is per key, not a prefix)
    bias = torch.randn(heads, 2 * seq - 1, generator=g).to(DEV) if with_bias else None
    q, k, qkv, allowed = _text_case(seq, heads, 3, key_mask, causal, g)
    buf = torch.full((3 * seq, heads * 64 + 64), AP.SENTINEL, device=DEV, dtype=torch.bfloat16)
    ops.attn_fwd_text(qkv, buf[:, :heads * 64], batch=3, heads=heads, seq=seq, scale=SCALE, bias=bias, key_mask=key_mask,
                      causal=causal)
    torch.cuda.synchronize()
    assert bool((buf[:, heads * 64:] == AP.SENTINEL).all())
    out = buf[:, :heads * 64].reshape(3, seq, heads * 64)
    p_ref, _ = AP.fwd_reference(q, k, allowed, SCALE, bias=bias)
    rep = AP.check_probs(f"text seq {seq} causal {causal} bias {with_bias}", out, p_ref, allowed,
                         AP.rel_bound_fwd(SCALE, AP.norm_product_max(q, k)))
    print(str(rep).splitlines()[0])
    assert rep.ok(), str(rep)


def test_text_all_zero_key_mask_gives_zero_rows():
    """pf_b200.h: a batch whose key mask is all zeros has no defined result and its rows are written as zeros (the host
    wrapper refuses such a mask, so this goes through the C ABI)."""
    _lib.require_device()
    seq, heads = 77, 3
    g = torch.Generator().manual_seed(3)
    key_mask = torch.ones(2, seq, dtype=torch.int32, device=DEV)
    key_mask[1] = 0
    q, k, qkv, allowed = _text_case(seq, heads, 2, key_mask, False, g)
    buf = torch.full((2 * seq, heads * 64), AP.SENTINEL, device=DEV, dtype=torch.bfloat16)
    d = AttnTextDesc()
    d.qkv, d.ld_qkv, d.out, d.ldo = qkv.data_ptr(), qkv.stride(0), buf.data_ptr(), buf.stride(0)
    d.batch, d.heads, d.seq, d.head_dim, d.scale = 2, heads, seq, 64, SCALE
    d.bias, d.key_mask, d.causal = None, key_mask.data_ptr(), 0
    _lib.check(_lib.load().pf_attn_fwd_text(C.byref(d), _lib.stream_ptr()), "pf_attn_fwd_text")
    torch.cuda.synchronize()
    out = buf.reshape(2, seq, heads * 64)
    assert bool((out[1] == 0).all())
    p_ref, _ = AP.fwd_reference(q[:1], k[:1], allowed[:1], SCALE)
    rep = AP.check_probs("text, the batch with keys", out[:1], p_ref, allowed[:1], AP.rel_bound_fwd(SCALE, AP.norm_product_max(q, k)))
    assert rep.ok(), str(rep)
