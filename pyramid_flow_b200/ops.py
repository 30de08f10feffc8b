"""Tensor-level wrappers over the C-ABI (one function per entry point in include/pf_b200.h).

Each wrapper validates dtypes/contiguity, passes raw pointers + the current stream, and raises on a non-zero status.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import (AttnBwdDesc, AttnDesc, AttnPackDesc, AttnTextDesc, AttnVarlenPackDesc, AttnVarlenUnpackDesc, ConvDesc,
                   ConvPackDesc, ConvWgradDesc, GemmDesc, GroupNormTrainDesc, PF_EPI_GATE_RESID, PF_EPI_GELU_BF16, PF_EPI_QKV_GELU,
                   PF_EPI_QKV_ROPE, PF_EPI_STORE_BF16, PF_EPI_STORE_F32)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _gemm_desc(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], epilogue: int, *,
               batches: int = 1, rows_per_batch: Optional[int] = None, row_begin: int = 0, row_count: Optional[int] = None,
               out: Optional[torch.Tensor] = None, ldo: Optional[int] = None, out_batch_rows: Optional[int] = None,
               out_row_begin: Optional[int] = None, out_col_begin: int = 0,
               gate: Optional[torch.Tensor] = None, gate_batch_stride: int = 0,
               q_out=None, k_out=None, v_out=None, rope=None, q_norm_w=None, k_norm_w=None, norm_eps: float = 1e-6,
               heads: int = 0, head_dim: int = 0, seq_len: int = 0, n_split: int = 0, kernel_variant: int = 0,
               peer: Optional[dict] = None) -> GemmDesc:
    """The pf_gemm_desc of one launch (operand dtypes are checked by the callers)."""
    assert a.is_cuda and w.is_cuda
    assert a.stride(-1) == 1 and w.is_contiguous()
    n, k = w.shape
    lda = a.stride(-2)
    if rows_per_batch is None:
        rows_per_batch = a.numel() // (a.shape[-1] * batches) if a.is_contiguous() else a.shape[-2]
    if row_count is None:
        row_count = rows_per_batch - row_begin
    d = GemmDesc()
    d.a, d.lda = a.data_ptr(), lda
    d.batches, d.rows_per_batch, d.row_begin, d.row_count = batches, rows_per_batch, row_begin, row_count
    d.w, d.n, d.k = w.data_ptr(), n, k
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
    d.bias = _ptr(bias)
    d.epilogue = epilogue
    d.out = _ptr(out)
    if out is not None:
        d.ldo = ldo if ldo is not None else out.stride(-2)
    d.out_batch_rows = out_batch_rows if out_batch_rows is not None else rows_per_batch
    d.out_row_begin = out_row_begin if out_row_begin is not None else row_begin
    d.out_col_begin = out_col_begin
    if gate is not None:
        assert gate.dtype == torch.float32
    d.gate, d.gate_batch_stride = _ptr(gate), gate_batch_stride
    d.q_out, d.k_out, d.v_out = _ptr(q_out), _ptr(k_out), _ptr(v_out)
    for t in (rope, q_norm_w, k_norm_w):
        if t is not None:
            assert t.dtype == torch.float32 and t.is_contiguous()
    d.rope, d.q_norm_w, d.k_norm_w = _ptr(rope), _ptr(q_norm_w), _ptr(k_norm_w)
    d.norm_eps = norm_eps
    d.heads, d.head_dim, d.seq_len, d.n_split = heads, head_dim, seq_len, n_split
    d.kernel_variant = kernel_variant
    if peer is not None:      # sequence parallel: QKV heads stored straight into the owning rank's buffer (pf_b200.h)
        for i, pp in enumerate(peer["peer_ptrs"]):
            d.peer_qkv[i] = pp
        d.peer_count, d.peer_heads = len(peer["peer_ptrs"]), peer["peer_heads"]
        d.peer_seq, d.peer_row0 = peer["peer_seq"], peer["peer_row0"]
    return d


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], epilogue: int, **kw) -> None:
    """epilogue(A . W^T + bias); see pf_gemm_bf16 in include/pf_b200.h for the addressing rules and `_gemm_desc` for the
    keyword arguments."""
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16
    d = _gemm_desc(a, w, bias, epilogue, **kw)
    _lib.check(_lib.load().pf_gemm_bf16(C.byref(d), _lib.stream_ptr()), "pf_gemm_bf16")


def gemm_fp8(a8: torch.Tensor, a_scale: torch.Tensor, w8: torch.Tensor, w_scale: torch.Tensor, bias: Optional[torch.Tensor],
             epilogue: int, **kw) -> None:
    """epilogue((A8 . W8^T) * a_scale[row] * w_scale[n] + bias) on e4m3 operands (pf_gemm_fp8); the keyword arguments are
    those of `gemm`.  a_scale: fp32 [batches, rows_per_batch] indexed like A's rows; w_scale: fp32 [n]."""
    assert a8.dtype == torch.float8_e4m3fn and w8.dtype == torch.float8_e4m3fn
    assert a_scale.dtype == torch.float32 and a_scale.is_contiguous() and w_scale.dtype == torch.float32
    assert w_scale.is_contiguous() and w_scale.numel() == w8.shape[0]
    d = _gemm_desc(a8, w8, bias, epilogue, **kw)
    assert a_scale.numel() >= d.batches * d.rows_per_batch
    _lib.check(_lib.load().pf_gemm_fp8(C.byref(d), a_scale.data_ptr(), w_scale.data_ptr(), _lib.stream_ptr()), "pf_gemm_fp8")


E4M3_MAX = 448.0


def quantize_weight_fp8(w: torch.Tensor):
    """Host quantiser of a weight [N, K] with one scale per output channel (include/pf_b200.h FP8 contract), from the values
    taken to fp32: -> (w8 float8_e4m3fn [N, K], scale fp32 [N]).  torch's cast does not saturate, but the scaled values stay
    within 448 (1 + 2^-23), which rounds to 448, so the bits are those of the device quantiser."""
    w = w.detach().float()
    amax = w.abs().amax(dim=1)
    # tensor / tensor divisions are IEEE; with a Python scalar torch may multiply by a reciprocal (two roundings)
    e4m3_max = torch.full_like(amax, E4M3_MAX)
    inv = torch.where(amax > 0, e4m3_max / amax, torch.zeros_like(amax))
    w8 = (w * inv[:, None]).to(torch.float8_e4m3fn).contiguous()
    return w8, (amax / e4m3_max).contiguous()


def linear_bf16(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, gelu: bool = False) -> torch.Tensor:
    """Convenience: y_bf16[M, N] = (gelu)(x[M, K] . w[N, K]^T + bias)."""
    m = x.shape[0]
    out = torch.empty(m, w.shape[0], dtype=torch.bfloat16, device=x.device)
    gemm(x, w, bias, PF_EPI_GELU_BF16 if gelu else PF_EPI_STORE_BF16, rows_per_batch=m, out=out)
    return out


def ln_modulate(x: torch.Tensor, y: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, mod_batch_stride: int, *,
                batches: int, rows_per_batch: int, row_begin: int, row_count: int, eps: float = 1e-6) -> None:
    assert x.dtype == torch.float32 and y.dtype == torch.bfloat16 and x.is_contiguous() and y.is_contiguous()
    dim = x.shape[-1]
    _lib.check(_lib.load().pf_ln_modulate(x.data_ptr(), y.data_ptr(), batches, rows_per_batch, row_begin, row_count,
                                          dim, shift.data_ptr(), scale.data_ptr(), mod_batch_stride, eps,
                                          _lib.stream_ptr()), "pf_ln_modulate")


def ln_modulate_fp8(x: torch.Tensor, y8: torch.Tensor, row_scale: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor,
                    mod_batch_stride: int, *, batches: int, rows_per_batch: int, row_begin: int, row_count: int,
                    eps: float = 1e-6) -> None:
    """ln_modulate with an e4m3 output y8 [.., dim] (row stride dim) and its per-row scales row_scale fp32
    [batches, rows_per_batch] (pf_ln_modulate_fp8)."""
    assert x.dtype == torch.float32 and x.is_contiguous() and y8.dtype == torch.float8_e4m3fn and y8.is_contiguous()
    assert row_scale.dtype == torch.float32 and row_scale.is_contiguous() and row_scale.numel() >= batches * rows_per_batch
    dim = x.shape[-1]
    assert y8.numel() >= batches * rows_per_batch * dim
    _lib.check(_lib.load().pf_ln_modulate_fp8(x.data_ptr(), y8.data_ptr(), row_scale.data_ptr(), batches, rows_per_batch,
                                              row_begin, row_count, dim, shift.data_ptr(), scale.data_ptr(),
                                              mod_batch_stride, eps, _lib.stream_ptr()), "pf_ln_modulate_fp8")


def quantize_rows_fp8(x: torch.Tensor, y8: torch.Tensor, row_scale: torch.Tensor, *, batches: int = 1,
                      rows_per_batch: Optional[int] = None, row_begin: int = 0, row_count: Optional[int] = None) -> None:
    """x bf16 [(batches,) rows, cols] (row stride x.stride(-2)) -> e4m3 y8 (same shape, row stride y8.stride(-2)) and
    row_scale fp32 [batches, rows_per_batch], for rows [row_begin, row_begin + row_count) of each batch (pf_quantize_rows_fp8)."""
    assert x.dtype == torch.bfloat16 and y8.dtype == torch.float8_e4m3fn and x.is_cuda and y8.is_cuda
    assert x.stride(-1) == 1 and y8.stride(-1) == 1 and x.shape[-1] == y8.shape[-1]
    assert row_scale.dtype == torch.float32 and row_scale.is_contiguous()
    if rows_per_batch is None:
        rows_per_batch = x.shape[-2]
    if row_count is None:
        row_count = rows_per_batch - row_begin
    assert row_scale.numel() >= batches * rows_per_batch
    _lib.check(_lib.load().pf_quantize_rows_fp8(x.data_ptr(), x.stride(-2), y8.data_ptr(), y8.stride(-2), row_scale.data_ptr(),
                                                batches, rows_per_batch, row_begin, row_count, x.shape[-1],
                                                _lib.stream_ptr()), "pf_quantize_rows_fp8")


def small_linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], y: torch.Tensor, *, act_in: int = 0,
                 act_out: int = 0, accumulate: bool = False, round_in_bf16: bool = False) -> None:
    assert x.dtype == torch.float32 and y.dtype == torch.float32 and w.dtype == torch.bfloat16
    assert x.is_contiguous() and w.is_contiguous() and y.is_contiguous()
    m, k = x.shape
    n = w.shape[0]
    assert w.shape[1] == k and y.shape == (m, n)
    _lib.check(_lib.load().pf_small_linear(x.data_ptr(), m, k, w.data_ptr(), _ptr(bias), n, y.data_ptr(), act_in,
                                           act_out, int(accumulate), int(round_in_bf16), _lib.stream_ptr()),
               "pf_small_linear")


def timestep_embedding(t: torch.Tensor, dim: int, round_bf16: bool = True) -> torch.Tensor:
    assert t.dtype == torch.float32 and t.is_contiguous()
    out = torch.empty(t.shape[0], dim, dtype=torch.float32, device=t.device)
    _lib.check(_lib.load().pf_timestep_embedding(t.data_ptr(), t.shape[0], dim, out.data_ptr(), int(round_bf16),
                                                 _lib.stream_ptr()), "pf_timestep_embedding")
    return out


def patchify(latent: torch.Tensor, tokens: torch.Tensor, rows_per_batch: int, tok_begin: int) -> None:
    assert latent.is_contiguous() and latent.dtype in (torch.float32, torch.bfloat16) and tokens.dtype == torch.bfloat16
    b, c, t, h, w = latent.shape
    _lib.check(_lib.load().pf_patchify(latent.data_ptr(), int(latent.dtype == torch.float32), b, c, t, h, w,
                                       tokens.data_ptr(), rows_per_batch, tok_begin, _lib.stream_ptr()), "pf_patchify")


def unpatchify(x: torch.Tensor, rows_per_batch: int, row_begin: int, out: torch.Tensor) -> None:
    assert x.dtype == torch.float32 and x.is_contiguous() and out.is_contiguous()
    b, c, t, h, w = out.shape
    _lib.check(_lib.load().pf_unpatchify(x.data_ptr(), rows_per_batch, row_begin, b, c, t, h, w, out.data_ptr(),
                                         int(out.dtype == torch.float32), _lib.stream_ptr()), "pf_unpatchify")


def cfg_euler_step(v2: torch.Tensor, guidance: float, dsigma: float, x: torch.Tensor, x_out: torch.Tensor) -> None:
    assert v2.dtype == torch.float32 and x.dtype == torch.float32 and x_out.dtype == torch.float32
    n = x.numel()
    assert v2.numel() == 2 * n
    _lib.check(_lib.load().pf_cfg_euler_step(v2.data_ptr(), guidance, dsigma, x.data_ptr(), x_out.data_ptr(), n,
                                             _lib.stream_ptr()), "pf_cfg_euler_step")


def stage_hop(x: torch.Tensor, z: torch.Tensor, alpha: float, beta: float, gamma: float) -> torch.Tensor:
    """x [b, c, t, h, w] (bf16/fp32) -> alpha * nearest_x2(x) + beta * block_noise(z), z iid normal fp32 [b, c, t, 2h, 2w]
    (pf_stage_hop; reference P:729-743 + P:697-703)."""
    import ctypes as C
    assert x.is_cuda and x.is_contiguous() and z.is_contiguous() and z.dtype == torch.float32
    assert x.dtype in (torch.float32, torch.bfloat16)
    b, c, t, h, w = x.shape
    assert tuple(z.shape) == (b, c, t, 2 * h, 2 * w)
    cov = torch.eye(4, dtype=torch.float64) * (1 + gamma) - torch.ones(4, 4, dtype=torch.float64) * gamma
    chol = torch.linalg.cholesky(cov).to(torch.float32).flatten().tolist()
    out = torch.empty(b, c, t, 2 * h, 2 * w, device=x.device, dtype=x.dtype)
    arr = (C.c_float * 16)(*chol)
    _lib.check(_lib.load().pf_stage_hop(x.data_ptr(), int(x.dtype == torch.float32), z.data_ptr(), out.data_ptr(), b * c * t, h, w,
                                        alpha, beta, arr, _lib.stream_ptr()), "pf_stage_hop")
    return out


def attn_build_schedule(seg: torch.Tensor, time: torch.Tensor):
    """seg/time: int32 CPU tensors [batch, seq] -> (schedule int32 CPU [batch, q_tiles, stride], allowed_pairs [batch])."""
    seg = seg.to(torch.int32).contiguous().cpu()
    time = time.to(torch.int32).contiguous().cpu()
    batch, seq = seg.shape
    lib = _lib.load()
    stride = lib.pf_attn_build_schedule(None, None, batch, seq, None, None)
    if stride < 0:
        _lib.check(stride, "pf_attn_build_schedule")
    qt = (seq + 127) // 128
    sched = torch.zeros(batch, qt, stride, dtype=torch.int32)
    pairs = torch.zeros(batch, dtype=torch.int64)
    rc = lib.pf_attn_build_schedule(seg.data_ptr(), time.data_ptr(), batch, seq, sched.data_ptr(), pairs.data_ptr())
    if rc < 0:
        _lib.check(rc, "pf_attn_build_schedule")
    return sched, pairs


class PairSchedule:
    """Schedule of pairs of q tiles: `sched` int32 [batch, n_pairs, stride] (pf_attn_build_pair_schedule),
    `mask_index` int32 [batch, n_pairs, 2 * stride] and `mask_bits` int32 [blocks, 128, 4] (pf_attn_build_pair_masks).
    `group3` (optional) = the same three tensors for groups of three q tiles (pf_attn_build_group_schedule / _masks), the
    schedule of groups of three q tiles."""

    def __init__(self, sched: torch.Tensor, mask_index: torch.Tensor, mask_bits: torch.Tensor,
                 group3: Optional["PairSchedule"] = None):
        self.sched, self.mask_index, self.mask_bits, self.group3 = sched, mask_index, mask_bits, group3

    def to(self, device) -> "PairSchedule":
        bits = self.mask_bits.to(device)
        g3 = self.group3
        if g3 is not None:     # the group schedule indexes the SAME block pool when it was built from this pair schedule
            g3 = PairSchedule(g3.sched.to(device), g3.mask_index.to(device), bits if g3.mask_bits is self.mask_bits else g3.mask_bits.to(device))
        return PairSchedule(self.sched.to(device), self.mask_index.to(device), bits, g3)

    def __getitem__(self, idx) -> "PairSchedule":          # batch slice (block indices are global: the bit pool is shared)
        assert isinstance(idx, slice)
        return PairSchedule(self.sched[idx], self.mask_index[idx], self.mask_bits,
                            None if self.group3 is None else self.group3[idx])


def attn_build_pair_schedule(sched: torch.Tensor, seq: int, seg: torch.Tensor, time: torch.Tensor) -> PairSchedule:
    """Tile schedule (int32 CPU [batch, q_tiles, stride]) + the seg/time ids -> PairSchedule (CPU tensors) of the q-tile pairs:
    merged kv lists of adjacent q tiles and the precomputed 128-bit row masks of their partial tiles."""
    sched = sched.to(torch.int32).contiguous().cpu()
    seg = seg.to(torch.int32).contiguous().cpu()
    time = time.to(torch.int32).contiguous().cpu()
    batch, qt, stride = sched.shape
    n_pairs = (qt + 1) // 2
    lib = _lib.load()
    ps = torch.zeros(batch, n_pairs, stride, dtype=torch.int32)
    _lib.check(lib.pf_attn_build_pair_schedule(sched.data_ptr(), batch, seq, stride, ps.data_ptr()), "pf_attn_build_pair_schedule")
    midx = torch.full((batch, n_pairs, 2 * stride), -1, dtype=torch.int32)
    n = lib.pf_attn_build_pair_masks(seg.data_ptr(), time.data_ptr(), ps.data_ptr(), batch, seq, stride, midx.data_ptr(), None, 0)
    if n < 0:
        _lib.check(int(n), "pf_attn_build_pair_masks")
    bits = torch.zeros(max(1, int(n)), 128, 4, dtype=torch.int32)
    n2 = lib.pf_attn_build_pair_masks(seg.data_ptr(), time.data_ptr(), ps.data_ptr(), batch, seq, stride, midx.data_ptr(),
                                      bits.data_ptr(), int(n))
    assert n2 == n
    pso = PairSchedule(ps, midx, bits)
    pso.group3 = attn_build_group_schedule(sched, seq, seg, time, 3, share=pso)
    return pso


def attn_build_group_schedule(sched: torch.Tensor, seq: int, seg: torch.Tensor, time: torch.Tensor, group: int = 3,
                              share: Optional[PairSchedule] = None) -> PairSchedule:
    """The pair schedule generalised to groups of `group` q tiles: sched int32 [batch, n_groups,
    stride] with entries (kv_tile << 8) | 2 flag bits per tile, mask_index [batch, n_groups, group * stride], mask_bits.
    `share` = the pair schedule of the same tile schedule: its block pool is reused (a block depends on (q tile, kv tile) only),
    no bits are built and `mask_bits` IS `share.mask_bits`."""
    sched = sched.to(torch.int32).contiguous().cpu()
    seg = seg.to(torch.int32).contiguous().cpu()
    time = time.to(torch.int32).contiguous().cpu()
    batch, qt, stride = sched.shape
    n_groups = (qt + group - 1) // group
    lib = _lib.load()
    gs = torch.zeros(batch, n_groups, stride, dtype=torch.int32)
    _lib.check(lib.pf_attn_build_group_schedule(sched.data_ptr(), batch, seq, stride, group, gs.data_ptr()), "pf_attn_build_group_schedule")
    midx = torch.full((batch, n_groups, group * stride), -1, dtype=torch.int32)
    if share is not None:
        assert share.sched.shape[-1] == stride and share.sched.is_contiguous() and share.mask_index.is_contiguous()
        n = lib.pf_attn_build_group_masks(seg.data_ptr(), time.data_ptr(), gs.data_ptr(), batch, seq, stride, group, midx.data_ptr(),
                                          None, 0, share.sched.data_ptr(), share.mask_index.data_ptr())
        if n < 0:
            _lib.check(int(n), "pf_attn_build_group_masks")
        assert n <= share.mask_bits.shape[0]
        return PairSchedule(gs, midx, share.mask_bits)
    n = lib.pf_attn_build_group_masks(seg.data_ptr(), time.data_ptr(), gs.data_ptr(), batch, seq, stride, group, midx.data_ptr(), None, 0,
                                      None, None)
    if n < 0:
        _lib.check(int(n), "pf_attn_build_group_masks")
    bits = torch.zeros(max(1, int(n)), 128, 4, dtype=torch.int32)
    n2 = lib.pf_attn_build_group_masks(seg.data_ptr(), time.data_ptr(), gs.data_ptr(), batch, seq, stride, group, midx.data_ptr(),
                                       bits.data_ptr(), int(n), None, None)
    assert n2 == n
    return PairSchedule(gs, midx, bits)


def attn_build_kv_schedule(sched: torch.Tensor, seq: int) -> torch.Tensor:
    """Tile schedule (int32 CPU [batch, q_tiles, stride], attn_build_schedule) -> its kv-major transpose, int32 CPU
    [batch, kv_tiles, stride]: per kv tile [count, (q_tile << 1) | needs_mask, ...] (pf_attn_build_kv_schedule)."""
    sched = sched.to(torch.int32).contiguous().cpu()
    batch, tiles, stride = sched.shape
    out = torch.zeros(batch, tiles, stride, dtype=torch.int32)
    _lib.check(_lib.load().pf_attn_build_kv_schedule(sched.data_ptr(), batch, seq, stride, out.data_ptr()),
               "pf_attn_build_kv_schedule")
    return out


def attn_fwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, seg: torch.Tensor,
             time: torch.Tensor, sched: torch.Tensor, scale: float, variant: int = 0, q_row_begin: int = 0,
             pair_sched: Optional[PairSchedule] = None, ldo: Optional[int] = None, peer: Optional[dict] = None,
             lse: Optional[torch.Tensor] = None) -> None:
    """q,k,v bf16 [B,H,S,64]; out bf16 [B,S,*] (row stride = out.stride(1)); seg/time/sched int32 on device.
    Only q rows >= q_row_begin (multiple of 128) are computed; other rows of `out` are left untouched.
    lse: optional fp32 [B,H,S], filled with each row's natural-log log-sum-exp of the scaled scores (for attn_bwd)."""
    assert q.dtype == torch.bfloat16 and q.is_contiguous() and k.is_contiguous() and v.is_contiguous()
    b, h, s, hd = q.shape
    d = AttnDesc()
    d.q, d.k, d.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    if out is not None:
        d.out = out.data_ptr()
        d.ldo = out.stride(-2)
    if ldo is not None:
        d.ldo = ldo
    if peer is not None:      # sequence parallel: output rows stored straight into the owning rank's buffer (pf_b200.h)
        for i, pp in enumerate(peer["peer_ptrs"]):
            d.peer_out[i] = pp
        d.peer_count, d.peer_chunk_rows, d.peer_col_begin = len(peer["peer_ptrs"]), peer["peer_chunk_rows"], peer["peer_col_begin"]
    d.batch, d.heads, d.seq, d.head_dim = b, h, s, hd
    d.scale = scale
    d.seg, d.time, d.tile_sched = seg.data_ptr(), time.data_ptr(), sched.data_ptr()
    d.sched_stride = sched.shape[-1]
    d.variant = variant
    d.q_row_begin = q_row_begin
    if pair_sched is not None:
        assert pair_sched.sched.dtype == torch.int32 and pair_sched.sched.shape[-1] == sched.shape[-1]
        assert pair_sched.sched.is_contiguous() and pair_sched.mask_index.is_contiguous() and pair_sched.mask_bits.is_contiguous()
        d.pair_sched = pair_sched.sched.data_ptr()
        d.pair_mask_index = pair_sched.mask_index.data_ptr()
        d.pair_mask_bits = pair_sched.mask_bits.data_ptr()
        g3 = pair_sched.group3
        if g3 is not None:
            assert g3.sched.is_contiguous() and g3.mask_index.is_contiguous() and g3.mask_bits.is_contiguous()
            assert g3.sched.shape[-1] == sched.shape[-1]
            d.group_sched, d.group_mask_index, d.group_mask_bits = g3.sched.data_ptr(), g3.mask_index.data_ptr(), g3.mask_bits.data_ptr()
    if lse is not None:
        assert lse.dtype == torch.float32 and lse.is_contiguous() and tuple(lse.shape) == (b, h, s)
        d.lse = lse.data_ptr()
    _lib.check(_lib.load().pf_attn_fwd_masked(C.byref(d), _lib.stream_ptr()), "pf_attn_fwd_masked")


def attn_bwd_rows_ok(t: torch.Tensor) -> bool:
    """Whether a bf16 [B, S, >=H*64] tensor can be handed to attn_bwd as it is (pf_attn_bwd_masked's layout rules: unit
    column stride, row and batch strides multiples of 8 elements, 16-byte aligned)."""
    return (t.dtype == torch.bfloat16 and t.ndim == 3 and t.stride(2) == 1 and t.stride(1) % 8 == 0 and t.stride(0) % 8 == 0
            and t.stride(1) >= t.shape[2] and t.stride(0) > 0 and t.data_ptr() % 16 == 0)


def attn_bwd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor,
             seg: torch.Tensor, time: torch.Tensor, sched: torch.Tensor, kv_sched: torch.Tensor, scale: float,
             dq: torch.Tensor, dk: torch.Tensor, dv: torch.Tensor, delta: Optional[torch.Tensor] = None) -> None:
    """Gradients of attn_fwd (pf_attn_bwd_masked): q,k,v,dq,dk,dv bf16 [B,H,S,64]; out/dout bf16 [B,S,>=H*64], any views
    that satisfy attn_bwd_rows_ok (their row and batch strides are passed); lse fp32 [B,H,S] from attn_fwd;
    seg/time/sched/kv_sched int32 on the device."""
    b, h, s, hd = q.shape
    for t in (q, k, v, dq, dk, dv):
        assert t.dtype == torch.bfloat16 and t.is_cuda and t.is_contiguous() and tuple(t.shape) == (b, h, s, hd)
    for t in (out, dout):
        assert t.is_cuda and tuple(t.shape[:2]) == (b, s) and t.shape[2] >= h * hd, (tuple(t.shape), (b, s, h * hd))
        assert attn_bwd_rows_ok(t), f"attn_bwd: layout {tuple(t.stride())} not supported, pass a contiguous copy"
    assert lse.dtype == torch.float32 and lse.is_contiguous() and tuple(lse.shape) == (b, h, s)
    assert sched.shape == kv_sched.shape and sched.dtype == torch.int32 and kv_sched.dtype == torch.int32
    if delta is None:
        delta = torch.empty(b, h, s, dtype=torch.float32, device=q.device)
    d = AttnBwdDesc()
    d.q, d.k, d.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    d.out, d.ldo, d.out_batch_stride = out.data_ptr(), out.stride(1), out.stride(0)
    d.dout, d.lddo, d.dout_batch_stride = dout.data_ptr(), dout.stride(1), dout.stride(0)
    d.lse = lse.data_ptr()
    d.batch, d.heads, d.seq, d.head_dim = b, h, s, hd
    d.scale = scale
    d.seg, d.time, d.tile_sched, d.kv_sched = seg.data_ptr(), time.data_ptr(), sched.data_ptr(), kv_sched.data_ptr()
    d.sched_stride = sched.shape[-1]
    d.delta, d.dq, d.dk, d.dv = delta.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr()
    _lib.check(_lib.load().pf_attn_bwd_masked(C.byref(d), _lib.stream_ptr()), "pf_attn_bwd_masked")


def attn_pack_source_ok(t: torch.Tensor) -> bool:
    """Whether a [B, S, H, 64] q / k / v view can be read (or, as a gradient, written) by the stage pack as it is
    (pf_attn_stage_pack's layout rules: bf16 or fp32, unit column stride, other strides positive multiples of 8 elements,
    16-byte aligned)."""
    return (t.dtype in (torch.bfloat16, torch.float32) and t.ndim == 4 and t.shape[-1] == 64 and t.stride(3) == 1
            and all(st > 0 and st % 8 == 0 for st in t.stride()[:3]) and t.data_ptr() % 16 == 0)


def _pack_desc(video, text, freqs, packed, row0: int, stage: int, n_stages: int) -> AttnPackDesc:
    b, h, seq, hd = packed[0].shape
    text_len = 0 if text is None else text[0].shape[1]
    for t in packed:
        assert t.dtype == torch.bfloat16 and t.is_cuda and t.is_contiguous() and tuple(t.shape) == (b, h, seq, hd)
    d = AttnPackDesc()
    d.batch, d.heads, d.head_dim, d.text_len = b, h, hd, text_len
    d.rows, d.row0, d.src_rows = seq - text_len, row0, video[0].shape[1]
    d.n_stages, d.stage = n_stages, stage
    for i, t in enumerate(video):
        assert t.is_cuda and t.shape[0] == b and t.shape[2:] == (h, hd) and t.shape[1] == d.src_rows and attn_pack_source_ok(t), \
            (tuple(t.shape), t.stride(), t.dtype)
        d.video[i], d.video_f32[i] = t.data_ptr(), int(t.dtype == torch.float32)
        for j in range(3):
            d.video_strides[i][j] = t.stride(j)
    if text is not None:
        for i, t in enumerate(text):
            assert t.is_cuda and tuple(t.shape) == (b * n_stages, text_len, h, hd) and attn_pack_source_ok(t), \
                (tuple(t.shape), t.stride(), t.dtype)
            d.text[i], d.text_f32[i] = t.data_ptr(), int(t.dtype == torch.float32)
            for j in range(3):
                d.text_strides[i][j] = t.stride(j)
    if freqs is not None:
        assert freqs.dtype == torch.float32 and freqs.is_cuda and freqs.numel() == b * seq * 128, tuple(freqs.shape)
        f = freqs.reshape(b, seq, 128)
        assert f.stride(2) == 1
        d.freqs, d.freqs_batch_stride, d.freqs_row_stride = f.data_ptr(), f.stride(0), f.stride(1)
    for i, t in enumerate(packed):
        d.packed[i] = t.data_ptr()
    return d


def attn_stage_pack(video, text, freqs: Optional[torch.Tensor], packed, *, row0: int, stage: int = 0, n_stages: int = 1) -> None:
    """One stage's head-major q, k, v for attn_fwd / attn_bwd (pf_attn_stage_pack): packed = (q, k, v) bf16 [B, H, T + L, 64]
    from the text rows of encoder row b * n_stages + stage of text = (q, k, v) [B * n_stages, T, H, 64] (None: T = 0), then
    rows [row0, row0 + L) of video = (q, k, v) [B, S_total, H, 64]; sources bf16 or fp32 views satisfying attn_pack_source_ok.
    freqs: fp32 [B, T + L, (1,) 32, 2, 2] or None; applied to q and k as the reference's apply_rope does."""
    d = _pack_desc(video, text, freqs, packed, row0, stage, n_stages)
    _lib.check(_lib.load().pf_attn_stage_pack(C.byref(d), _lib.stream_ptr()), "pf_attn_stage_pack")


def attn_stage_pack_bwd(video_grad, text_grad, freqs: Optional[torch.Tensor], packed_grad, *, row0: int, stage: int = 0,
                        n_stages: int = 1) -> None:
    """The gradient inverse of attn_stage_pack (pf_attn_stage_pack_bwd): reads packed_grad = (dq, dk, dv) and writes the
    stage's rows of video_grad / text_grad (same shapes and rules as the sources, each in its own dtype)."""
    d = _pack_desc(video_grad, text_grad, freqs, packed_grad, row0, stage, n_stages)
    _lib.check(_lib.load().pf_attn_stage_pack_bwd(C.byref(d), _lib.stream_ptr()), "pf_attn_stage_pack_bwd")


def _varlen_layout(layout, *, batch: int, heads: int, text_len: int, src_rows: int, stage_len, stage_row0, row_map, pad_map) -> None:
    assert 1 <= len(stage_len) == len(stage_row0) <= _lib.VARLEN_MAX_STAGES, (list(stage_len), list(stage_row0))
    for m in (row_map, pad_map):
        assert m.dtype == torch.int32 and m.is_cuda and m.is_contiguous() and m.ndim == 1
    assert pad_map.numel() == batch * sum(stage_len), (pad_map.numel(), batch, list(stage_len))
    layout.batch, layout.heads, layout.head_dim, layout.text_len, layout.src_rows = batch, heads, 64, text_len, src_rows
    layout.n_stages, layout.total = len(stage_len), row_map.numel()
    for i, (n, r0) in enumerate(zip(stage_len, stage_row0)):
        layout.stage_len[i], layout.stage_row0[i] = n, r0
    layout.row_map, layout.pad_map = row_map.data_ptr(), pad_map.data_ptr()


def attn_varlen_pack(video, text, freqs, packed, *, stage_len, stage_row0, row_map: torch.Tensor, pad_map: torch.Tensor,
                     bwd: bool = False) -> None:
    """Every stage of a call site packed without its dropped rows (pf_attn_varlen_pack, or with bwd=True its gradient inverse
    pf_attn_varlen_pack_bwd): packed = (q, k, v) bf16 [1, H, total, 64]; video = (q, k, v) [B, src_rows, H, 64], text = (q, k,
    v) [B * n_stages, T, H, 64] or None, bf16 / fp32 views satisfying attn_pack_source_ok (the gradients to write, with bwd);
    freqs: per stage fp32 [B, stage_len[i], (1,) 32, 2, 2] or None; row_map / pad_map int32 on the device (pf_b200.h)."""
    b, src_rows, h, hd = video[0].shape
    total = row_map.numel()
    text_len = 0 if text is None else text[0].shape[1]
    d = AttnVarlenPackDesc()
    _varlen_layout(d.layout, batch=b, heads=h, text_len=text_len, src_rows=src_rows, stage_len=stage_len, stage_row0=stage_row0,
                   row_map=row_map, pad_map=pad_map)
    for i, t in enumerate(packed):
        assert t.dtype == torch.bfloat16 and t.is_cuda and t.is_contiguous() and tuple(t.shape) == (1, h, total, hd)
        d.packed[i] = t.data_ptr()
    for i, t in enumerate(video):
        assert t.is_cuda and tuple(t.shape) == (b, src_rows, h, hd) and attn_pack_source_ok(t), (tuple(t.shape), t.stride(), t.dtype)
        d.video[i], d.video_f32[i] = t.data_ptr(), int(t.dtype == torch.float32)
        for j in range(3):
            d.video_strides[i][j] = t.stride(j)
    if text is not None:
        for i, t in enumerate(text):
            assert t.is_cuda and tuple(t.shape) == (b * len(stage_len), text_len, h, hd) and attn_pack_source_ok(t), \
                (tuple(t.shape), t.stride(), t.dtype)
            d.text[i], d.text_f32[i] = t.data_ptr(), int(t.dtype == torch.float32)
            for j in range(3):
                d.text_strides[i][j] = t.stride(j)
    if freqs is not None:
        for i, (f, n) in enumerate(zip(freqs, stage_len)):
            assert f.dtype == torch.float32 and f.is_cuda and f.numel() == b * n * 128, (i, tuple(f.shape), n)
            f = f.reshape(b, n, 128)
            assert f.stride(2) == 1
            d.freqs[i], d.freqs_batch_stride[i], d.freqs_row_stride[i] = f.data_ptr(), f.stride(0), f.stride(1)
    name = "pf_attn_varlen_pack_bwd" if bwd else "pf_attn_varlen_pack"
    _lib.check(getattr(_lib.load(), name)(C.byref(d), _lib.stream_ptr()), name)


def attn_varlen_rows_ok(t: torch.Tensor) -> bool:
    """Whether a [B, S, H*64] output (or output gradient) view can be written (read) by the varlen unpack as it is: bf16 or
    fp32, unit column stride, batch and row strides positive multiples of 8 elements, 16-byte aligned."""
    return (t.dtype in (torch.bfloat16, torch.float32) and t.ndim == 3 and t.stride(2) == 1 and t.stride(0) > 0
            and t.stride(0) % 8 == 0 and t.stride(1) % 8 == 0 and t.stride(1) >= t.shape[2] and t.data_ptr() % 16 == 0)


def attn_varlen_unpack(video, text, packed: torch.Tensor, *, stage_len, stage_row0, row_map: torch.Tensor, pad_map: torch.Tensor,
                       bwd: bool = False) -> None:
    """The attention output packed bf16 [1, total, H*64] scattered into video [B, src_rows, H*64] and text [B * n_stages, T,
    H*64] (or None), zeros for dropped rows (pf_attn_varlen_unpack); with bwd=True the gradients video / text gathered into
    packed (pf_attn_varlen_unpack_bwd).  video / text: bf16 or fp32 views satisfying attn_varlen_rows_ok."""
    b, src_rows, width = video.shape
    h = width // 64
    assert width == h * 64 and packed.dtype == torch.bfloat16 and packed.is_cuda and packed.stride(-1) == 1
    assert tuple(packed.shape) == (1, row_map.numel(), width), (tuple(packed.shape), row_map.numel(), width)
    text_len = 0 if text is None else text.shape[1]
    d = AttnVarlenUnpackDesc()
    _varlen_layout(d.layout, batch=b, heads=h, text_len=text_len, src_rows=src_rows, stage_len=stage_len, stage_row0=stage_row0,
                   row_map=row_map, pad_map=pad_map)
    assert video.is_cuda and attn_varlen_rows_ok(video), (tuple(video.shape), video.stride(), video.dtype)
    d.video, d.video_strides[0], d.video_strides[1], d.video_f32 = video.data_ptr(), video.stride(0), video.stride(1), int(
        video.dtype == torch.float32)
    if text is not None:
        assert text.is_cuda and tuple(text.shape) == (b * len(stage_len), text_len, width) and attn_varlen_rows_ok(text), \
            (tuple(text.shape), text.stride(), text.dtype)
        d.text, d.text_strides[0], d.text_strides[1], d.text_f32 = text.data_ptr(), text.stride(0), text.stride(1), int(
            text.dtype == torch.float32)
    d.packed, d.ld_packed = packed.data_ptr(), packed.stride(1)
    name = "pf_attn_varlen_unpack_bwd" if bwd else "pf_attn_varlen_unpack"
    _lib.check(getattr(_lib.load(), name)(C.byref(d), _lib.stream_ptr()), name)


def attn_fwd_text(qkv: torch.Tensor, out: torch.Tensor, *, batch: int, heads: int, seq: int, scale: float,
                  bias: Optional[torch.Tensor] = None, key_mask: Optional[torch.Tensor] = None, causal: bool = False) -> None:
    """Short-sequence attention of the text encoders (pf_attn_fwd_text): qkv bf16 [batch * seq, >= 3 * heads * 64] (q | k | v
    per head, row stride qkv.stride(0)) -> out bf16 [batch * seq, >= heads * 64].  bias fp32 [heads, 2 seq - 1] (T5 relative
    position bias as a Toeplitz table), key_mask int32 [batch, seq] on the device (0 removes the key for every query)."""
    assert qkv.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and qkv.is_cuda and out.is_cuda
    assert qkv.stride(-1) == 1 and out.stride(-1) == 1 and qkv.shape[0] == batch * seq and out.shape[0] == batch * seq
    d = AttnTextDesc()
    d.qkv, d.ld_qkv, d.out, d.ldo = qkv.data_ptr(), qkv.stride(0), out.data_ptr(), out.stride(0)
    d.batch, d.heads, d.seq, d.head_dim = batch, heads, seq, 64
    d.scale = scale
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous() and tuple(bias.shape) == (heads, 2 * seq - 1)
    if key_mask is not None:
        assert key_mask.dtype == torch.int32 and key_mask.is_contiguous() and tuple(key_mask.shape) == (batch, seq)
    d.bias, d.key_mask, d.causal = _ptr(bias), _ptr(key_mask), int(causal)
    _lib.check(_lib.load().pf_attn_fwd_text(C.byref(d), _lib.stream_ptr()), "pf_attn_fwd_text")


def rms_norm_rows(x: torch.Tensor, y: torch.Tensor, w: torch.Tensor, *, batches: int = 1, rows_per_batch: Optional[int] = None,
                  row_begin: int = 0, row_count: Optional[int] = None, eps: float = 1e-6) -> None:
    """T5LayerNorm: x fp32 [.., dim] -> y bf16 (same row layout) = x * rsqrt(mean(x^2) + eps) * w (pf_rms_norm_rows)."""
    assert x.dtype == torch.float32 and y.dtype == torch.bfloat16 and w.dtype == torch.float32
    assert x.is_contiguous() and y.is_contiguous() and w.is_contiguous() and x.shape == y.shape
    dim = x.shape[-1]
    if rows_per_batch is None:
        rows_per_batch = x.numel() // (dim * batches)
    if row_count is None:
        row_count = rows_per_batch - row_begin
    _lib.check(_lib.load().pf_rms_norm_rows(x.data_ptr(), y.data_ptr(), w.data_ptr(), batches, rows_per_batch, row_begin, row_count,
                                            dim, eps, _lib.stream_ptr()), "pf_rms_norm_rows")


def embed_tokens(ids: torch.Tensor, table: torch.Tensor, out: torch.Tensor, *, rows_per_batch: int,
                 pos_table: Optional[torch.Tensor] = None) -> None:
    """out fp32 [rows, dim] = table[ids] (+ pos_table[row % rows_per_batch]) (pf_embed_tokens); ids int32 [rows] on the device."""
    assert ids.dtype == torch.int32 and ids.is_contiguous() and table.dtype == torch.bfloat16 and table.is_contiguous()
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape == (ids.numel(), table.shape[1])
    max_pos = 0
    if pos_table is not None:
        assert pos_table.dtype == torch.bfloat16 and pos_table.is_contiguous() and pos_table.shape[1] == table.shape[1]
        max_pos = pos_table.shape[0]
    _lib.check(_lib.load().pf_embed_tokens(ids.data_ptr(), ids.numel(), rows_per_batch, table.data_ptr(), table.shape[0],
                                           table.shape[1], _ptr(pos_table), max_pos, out.data_ptr(), _lib.stream_ptr()),
               "pf_embed_tokens")


def conv3d_pack(src: torch.Tensor, dst: torch.Tensor, *, t_offset: int, dil=(1, 1, 1),
                bias_grad: Optional[torch.Tensor] = None) -> None:
    """src [B, C, T, H, W] (bf16 or fp32, any strides) -> dst channels-last bf16 [B, T_total, H*dil_h, W*dil_w, Cpad]
    (pf_conv3d_pack): voxel (t, h, w) at (t_offset + t*dil_t, h*dil_h, w*dil_w), zeros elsewhere; bias_grad fp32 [C] = sum of
    src over every axis but C."""
    assert src.dtype in (torch.bfloat16, torch.float32) and src.dim() == 5 and src.is_cuda
    assert dst.dtype == torch.bfloat16 and dst.is_contiguous() and dst.dim() == 5
    b, c, t, h, w = src.shape
    d = ConvPackDesc()
    d.src, d.src_f32 = src.data_ptr(), int(src.dtype == torch.float32)
    d.b, d.c, d.t, d.h, d.w = b, c, t, h, w
    for i, s in enumerate(src.stride()):
        d.strides[i] = s
    d.dst, d.cpad, d.t_total, d.t_offset = dst.data_ptr(), dst.shape[-1], dst.shape[1], t_offset
    d.dil_t, d.dil_h, d.dil_w = dil
    assert tuple(dst.shape[2:4]) == (h * dil[1], w * dil[2]) and dst.shape[0] == b
    ws = None
    if bias_grad is not None:
        assert bias_grad.dtype == torch.float32 and bias_grad.is_contiguous() and bias_grad.numel() == c
        rows = b * t * h
        ws = torch.empty((rows + min(rows, 128)) * dst.shape[-1], device=src.device, dtype=torch.float32)
        d.bias_grad, d.workspace, d.workspace_floats = bias_grad.data_ptr(), ws.data_ptr(), ws.numel()
    _lib.check(_lib.load().pf_conv3d_pack(C.byref(d), _lib.stream_ptr()), "pf_conv3d_pack")


def causal_conv3d(x: torch.Tensor, wgt: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor, *, kernel, stride=(1, 1, 1),
                  store_channels: Optional[int] = None) -> None:
    """pf_causal_conv3d, plain store.  x bf16 [B, (t-1)*st + kt, h*sh, w*sw, cin_p] (packed, causal frames in front);
    wgt bf16 [cout_p, taps*cin_p]; bias fp32 [cout_p] or None; out bf16 / fp32 [B, t, h, w, out_c] (the output dims)."""
    kt, kh, kw = kernel
    st, sh, sw = stride
    b, t, h, w, out_c = out.shape
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and wgt.dtype == torch.bfloat16 and wgt.is_contiguous()
    assert out.is_contiguous() and out.dtype in (torch.bfloat16, torch.float32)
    assert tuple(x.shape[:4]) == (b, (t - 1) * st + kt, h * sh, w * sw), (tuple(x.shape), tuple(out.shape), stride)
    assert wgt.shape[1] == kt * kh * kw * x.shape[-1]
    assert bias is None or (bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == wgt.shape[0])
    d = ConvDesc()
    d.x, d.b, d.t, d.h, d.w, d.cin = x.data_ptr(), b, t, h, w, x.shape[-1]
    d.wgt, d.bias = wgt.data_ptr(), _ptr(bias)
    d.cout, d.kt, d.kh, d.kw = wgt.shape[0], kt, kh, kw
    d.store_mode, d.out, d.out_f32 = 0, out.data_ptr(), int(out.dtype == torch.float32)
    d.out_t_total, d.out_t_offset, d.out_c = t, 0, out_c
    d.store_channels = out_c if store_channels is None else store_channels
    d.stride_t, d.stride_h, d.stride_w = st, sh, sw
    _lib.check(_lib.load().pf_causal_conv3d(C.byref(d), _lib.stream_ptr()), "pf_causal_conv3d")


def conv3d_wgrad(xp: torch.Tensor, dyp: torch.Tensor, dw: torch.Tensor, *, out_shape, stride=(1, 1, 1)) -> None:
    """dw fp32 [Cout, Cin, kt, kh, kw] (pf_conv3d_wgrad) from the packed forward input xp bf16 [B, (t-1)*st + kt, h*sh, w*sw,
    cin_p] and the packed gradient dyp bf16 [B, T_total, h*sh, w*sw, cout_p]; out_shape = the output's (t, h, w)."""
    t, h, w = out_shape
    cout, cin, kt, kh, kw = dw.shape
    assert xp.dtype == dyp.dtype == torch.bfloat16 and xp.is_contiguous() and dyp.is_contiguous()
    assert dw.dtype == torch.float32 and dw.is_contiguous() and xp.shape[0] == dyp.shape[0]
    d = ConvWgradDesc()
    d.x, d.dy, d.dy_t_total = xp.data_ptr(), dyp.data_ptr(), dyp.shape[1]
    d.b, d.t, d.h, d.w = xp.shape[0], t, h, w
    d.cin, d.cout, d.cin_real, d.cout_real = xp.shape[-1], dyp.shape[-1], cin, cout
    d.kt, d.kh, d.kw = kt, kh, kw
    d.stride_t, d.stride_h, d.stride_w = stride
    lib = _lib.load()
    need = int(lib.pf_conv3d_wgrad_workspace(C.byref(d)))
    if need < 0:
        raise RuntimeError(f"libpf_b200 pf_conv3d_wgrad_workspace failed: {lib.pf_last_error().decode()}")
    ws = torch.empty(need, device=dw.device, dtype=torch.float32)
    d.dw, d.workspace, d.workspace_floats = dw.data_ptr(), ws.data_ptr(), need
    _lib.check(lib.pf_conv3d_wgrad(C.byref(d), _lib.stream_ptr()), "pf_conv3d_wgrad")


def groupnorm_form(x: torch.Tensor) -> Optional[str]:
    """The layout form pf_groupnorm_train_* read x [B, C, T, H, W] in: "channel" (channels_last_3d, every 8-channel vector
    16-byte aligned), "plane" (unit-stride (h, w) planes, e.g. NCDHW) or None (neither: the kernels refuse it).  Strides
    of size-1 axes are ignored, as in the library."""
    b, c, t, h, w = x.shape
    s = [0 if n == 1 else st for n, st in zip(x.shape, x.stride())]
    if (s[1] == 1 and (w == 1 or s[4] == c) and (h == 1 or s[3] == w * c) and s[0] % 8 == 0 and s[2] % 8 == 0
            and x.data_ptr() % 16 == 0):
        return "channel"
    if (w == 1 or s[4] == 1) and (h == 1 or s[3] == w):
        return "plane"
    return None


def _groupnorm_desc(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, stats: torch.Tensor, groups: int, eps: float,
                    silu: bool) -> GroupNormTrainDesc:
    assert x.dtype in (torch.bfloat16, torch.float32) and x.dim() == 5 and x.is_cuda
    assert gamma.dtype == beta.dtype == stats.dtype == torch.float32 and gamma.is_contiguous() and beta.is_contiguous()
    b, c, t, h, w = x.shape
    assert gamma.numel() == beta.numel() == c and stats.is_contiguous() and stats.numel() == b * t * groups * 2
    d = GroupNormTrainDesc()
    d.x, d.x_f32 = x.data_ptr(), int(x.dtype == torch.float32)
    d.b, d.c, d.t, d.h, d.w = b, c, t, h, w
    for i, st in enumerate(x.stride()):
        d.x_strides[i] = st
    d.groups, d.eps, d.silu = groups, eps, int(silu)
    d.gamma, d.beta, d.stats = gamma.data_ptr(), beta.data_ptr(), stats.data_ptr()
    return d


def _groupnorm_workspace(d: GroupNormTrainDesc, device) -> torch.Tensor:
    lib = _lib.load()
    need = int(lib.pf_groupnorm_train_workspace(C.byref(d)))
    if need < 0:
        raise RuntimeError(f"libpf_b200 pf_groupnorm_train_workspace failed: {lib.pf_last_error().decode()}")
    ws = torch.empty(need, device=device, dtype=torch.float32)
    d.workspace, d.workspace_floats = ws.data_ptr(), need
    return ws


def _dense_in_form(t: torch.Tensor, form: str) -> bool:
    if form == "channel":
        return t.permute(0, 2, 3, 4, 1).is_contiguous()
    return t.is_contiguous()


def groupnorm_train_fwd(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, stats: torch.Tensor, y: torch.Tensor, *,
                        groups: int, eps: float, silu: bool) -> None:
    """pf_groupnorm_train_fwd: stats fp32 [B*T, groups, 2] = per-frame (mean, rstd) of x [B, C, T, H, W] (bf16 / fp32, channel
    or plane form); y = act((x - mean) * rstd * gamma + beta), bf16 / fp32, x's shape, dense in x's form."""
    form = groupnorm_form(x)
    assert form is not None and y.shape == x.shape and y.dtype in (torch.bfloat16, torch.float32) and _dense_in_form(y, form)
    d = _groupnorm_desc(x, gamma, beta, stats, groups, eps, silu)
    d.y, d.y_f32 = y.data_ptr(), int(y.dtype == torch.float32)
    ws = _groupnorm_workspace(d, x.device)  # noqa: F841  (alive until the launch is queued)
    _lib.check(_lib.load().pf_groupnorm_train_fwd(C.byref(d), _lib.stream_ptr()), "pf_groupnorm_train_fwd")


def groupnorm_train_bwd(x: torch.Tensor, dy: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, stats: torch.Tensor,
                        dx: Optional[torch.Tensor], dgamma: Optional[torch.Tensor], dbeta: Optional[torch.Tensor], *,
                        groups: int, silu: bool) -> None:
    """pf_groupnorm_train_bwd: from dy (x's form, bf16 / fp32) and the forward's stats, dx (x's dtype, dense in x's form) and
    fp32 dgamma / dbeta [C]; any of the three may be None."""
    form = groupnorm_form(x)
    assert form is not None and dy.shape == x.shape and dy.dtype in (torch.bfloat16, torch.float32)
    assert dx is None or (dx.shape == x.shape and dx.dtype == x.dtype and _dense_in_form(dx, form))
    for p in (dgamma, dbeta):
        assert p is None or (p.dtype == torch.float32 and p.is_contiguous() and p.numel() == x.shape[1])
    d = _groupnorm_desc(x, gamma, beta, stats, groups, 0.0, silu)
    d.dy, d.dy_f32 = dy.data_ptr(), int(dy.dtype == torch.float32)
    for i, st in enumerate(dy.stride()):
        d.dy_strides[i] = st
    d.dx, d.dgamma, d.dbeta = _ptr(dx), _ptr(dgamma), _ptr(dbeta)
    ws = _groupnorm_workspace(d, x.device)  # noqa: F841
    _lib.check(_lib.load().pf_groupnorm_train_bwd(C.byref(d), _lib.stream_ptr()), "pf_groupnorm_train_bwd")
