"""Sequence / CFG parallel layout of the DiT step over N GPUs (one process per GPU, `torch.distributed`, NCCL on NVLink).

Follows the reference's sequence-parallel layout (trainer_misc/sp_utils.py:21-47 groups; Ulysses-style head<->sequence
all-to-all at the attention boundary, flux_modules/modeling_flux_block.py:266-325, 519-565 via trainer_misc/communicate.py)
with two changes the reference cannot make:
  * the CFG pair is split first (uncond / cond on separate halves of the world: no traffic until the velocity combine),
    so every rank runs batch 1 and the reference's `B % sp == 0` transposition trick (F:471-485) is not needed;
  * 30 heads do not divide by 4 or 8: heads are zero-padded to the next multiple of the SP degree (32 at sp=4, a 6.7 %
    attention overhead) instead of restricting miniFLUX to sp=2.
The joint sequence [text ; clips] is cut into `sp` contiguous chunks (all S of the 768p schedule are multiples of 8).

world = cfg_ways (2 if world >= 2 else 1) x sp;   rank -> (cfg_rank = rank // sp, sp_rank = rank % sp).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import torch
import torch.distributed as dist


@dataclass
class ParallelLayout:
    world: int
    rank: int
    cfg_ways: int
    sp: int
    cfg_rank: int
    sp_rank: int
    sp_group: Optional[object] = None    # ranks sharing a CFG branch
    cfg_group: Optional[object] = None   # the two ranks holding the same token chunk of the two branches

    @property
    def enabled(self) -> bool:
        return self.world > 1


def make_layout(world: Optional[int] = None, rank: Optional[int] = None, create_groups: bool = True) -> ParallelLayout:
    if world is None:
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        rank = dist.get_rank() if world > 1 else 0
    if world == 1:
        return ParallelLayout(1, 0, 1, 1, 0, 0)
    assert world % 2 == 0, "world size must be even (CFG pair is split first)"
    cfg_ways, sp = 2, world // 2
    lay = ParallelLayout(world, rank, cfg_ways, sp, rank // sp, rank % sp)
    if create_groups:
        # every rank must create every group (torch.distributed contract)
        for c in range(cfg_ways):
            g = dist.new_group(list(range(c * sp, (c + 1) * sp)))
            if c == lay.cfg_rank:
                lay.sp_group = g
        for s in range(sp):
            g = dist.new_group([s, sp + s])
            if s == lay.sp_rank:
                lay.cfg_group = g
    return lay


def padded_heads(heads: int, sp: int) -> int:
    return (heads + sp - 1) // sp * sp


def chunk_bounds(seq: int, sp: int, sp_rank: int) -> Tuple[int, int]:
    assert seq % sp == 0, f"sequence length {seq} must be divisible by the SP degree {sp}"
    n = seq // sp
    return sp_rank * n, (sp_rank + 1) * n


def peer_store_args(seq: int, sp: int, sp_rank: int, hp: int, qkv_ptrs, cat_ptrs):
    """The peer-store arguments of rank `sp_rank`'s launches (ops.gemm / ops.attn_fwd `peer=`), from the addresses of every sp
    rank's gathered q/k/v buffer (`qkv_ptrs`, bf16 [3, hp/sp, seq, 64]) and `cat` buffer (`cat_ptrs`, rows of this rank's
    chunk), in rank order.  The QKV epilogue stores head h of my chunk's rows into rank (h // Hg)'s gathered buffer at sequence
    position c0 + row; the attention epilogue stores each token chunk's rows of my head group straight into its owner's `cat`,
    at my head group's columns."""
    c0, c1 = chunk_bounds(seq, sp, sp_rank)
    hg = hp // sp
    peer_qkv = dict(peer_ptrs=list(qkv_ptrs), peer_heads=hg, peer_seq=seq, peer_row0=c0)
    peer_out = dict(peer_ptrs=list(cat_ptrs), peer_chunk_rows=c1 - c0, peer_col_begin=sp_rank * hg * 64)
    return peer_qkv, peer_out


def heads_to_sequence(x: torch.Tensor, lay: ParallelLayout) -> torch.Tensor:
    """Attention-boundary exchange #1 (reference B:285,295): x [Hp, S_local, hd] holds ALL (padded) heads of this rank's
    token chunk; returns [Hp/sp, S, hd] = this rank's head group over the WHOLE sequence.  One all_to_all_single."""
    hp, s_l, hd = x.shape
    hg = hp // lay.sp
    recv = torch.empty(lay.sp, hg, s_l, hd, dtype=x.dtype, device=x.device)
    dist.all_to_all_single(recv, x.view(lay.sp, hg, s_l, hd), group=lay.sp_group)
    # recv[src] = head group `sp_rank` of rank src's chunk -> concatenate the chunks along the sequence
    return recv.permute(1, 0, 2, 3).reshape(hg, lay.sp * s_l, hd)


def heads_to_sequence_qkv_begin(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, lay: ParallelLayout):
    """Start the three exchanges of one attention back to back (async on NCCL's stream); independent work — the single
    block's proj_mlp GEMM — can be launched on the compute stream before `heads_to_sequence_qkv_end` waits."""
    hp, s_l, hd = q.shape
    hg = hp // lay.sp
    recvs, works = [], []
    for x in (q, k, v):
        r = torch.empty(lay.sp, hg, s_l, hd, dtype=x.dtype, device=x.device)
        works.append(dist.all_to_all_single(r, x.view(lay.sp, hg, s_l, hd), group=lay.sp_group, async_op=True))
        recvs.append(r)
    return works, recvs, (hg, lay.sp * s_l, hd)


def heads_to_sequence_qkv_end(handle):
    works, recvs, shape = handle
    for w in works:
        w.wait()
    return tuple(r.permute(1, 0, 2, 3).reshape(shape) for r in recvs)


def heads_to_sequence_qkv(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, lay: ParallelLayout):
    return heads_to_sequence_qkv_end(heads_to_sequence_qkv_begin(q, k, v, lay))


def sequence_to_heads(o: torch.Tensor, lay: ParallelLayout) -> torch.Tensor:
    """Attention-boundary exchange #2 (reference B:314,321): o [S, Hg*hd] (this rank's head group, whole sequence, token
    major); returns [S_local, Hp*hd] = all heads for this rank's token chunk."""
    s, w = o.shape
    s_l = s // lay.sp
    recv = torch.empty(lay.sp, s_l, w, dtype=o.dtype, device=o.device)
    dist.all_to_all_single(recv, o.view(lay.sp, s_l, w), group=lay.sp_group)
    # recv[src] = head group src for my chunk -> heads concatenated along the feature axis
    return recv.permute(1, 0, 2).reshape(s_l, lay.sp * w)


# ----------------------------------------------------------------------------------------------------------------------
# Peer-memory exchange (default for sp > 1): the all-to-alls above become remote stores fused into the producing kernels
# (QKV GEMM epilogue, attention epilogue) over NVLink peer pointers + a flag barrier; see csrc/pf_peer.cu.
# ----------------------------------------------------------------------------------------------------------------------
class PeerBuffer:
    """One pf_peer_alloc buffer per rank of `ranks` (global ranks), mapped into every member: `.local` is this rank's buffer as
    a uint8 tensor, `.group()` the PfPeerGroup of mapped pointers in member order."""

    def __init__(self, nbytes: int, ranks, rank: int, gloo_group=None):
        import ctypes as C
        from . import _lib
        lib = _lib.load()
        self.nbytes = (int(nbytes) + 255) // 256 * 256
        self.ranks = list(ranks)
        self.my_index = self.ranks.index(rank)
        p = C.c_void_p()
        _lib.check(lib.pf_peer_alloc(self.nbytes, C.byref(p)), "pf_peer_alloc")
        self.ptr = p.value
        h = (C.c_ubyte * 64)()
        _lib.check(lib.pf_peer_export(self.ptr, h), "pf_peer_export")
        handles = [None] * dist.get_world_size()
        dist.all_gather_object(handles, (rank, bytes(h)), group=gloo_group)
        by_rank = dict(handles)
        self.ptrs = []
        for r in self.ranks:
            if r == rank:
                self.ptrs.append(self.ptr)
            else:
                q = C.c_void_p()
                hb = (C.c_ubyte * 64).from_buffer_copy(by_rank[r])
                _lib.check(lib.pf_peer_open(hb, C.byref(q)), f"pf_peer_open(rank {r})")
                self.ptrs.append(q.value)
        self.local = _as_tensor(self.ptr, self.nbytes)

    def close(self) -> None:
        from . import _lib
        lib = _lib.load()
        self.local = None
        for i, pp in enumerate(self.ptrs):
            if i != self.my_index:
                lib.pf_peer_close(pp)
        torch.cuda.synchronize()
        dist.barrier()                      # nobody frees while a peer still has the mapping open
        lib.pf_peer_free(self.ptr)
        self.ptrs = []

    def group(self, offset: int = 0):
        from ._lib import PeerGroup
        g = PeerGroup()
        for i, p in enumerate(self.ptrs):
            g.ptr[i] = p + offset
        g.n, g.my_index = len(self.ptrs), self.my_index
        return g

    def view(self, offset: int, shape, dtype) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= int(s)
        nb = n * torch.empty(0, dtype=dtype).element_size()
        assert offset % 256 == 0 and offset + nb <= self.nbytes
        return self.local[offset:offset + nb].view(dtype).view(*shape)


class _RawCuda:
    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


def _as_tensor(ptr: int, nbytes: int) -> torch.Tensor:
    return torch.as_tensor(_RawCuda(ptr, nbytes), device=torch.device("cuda", torch.cuda.current_device()))


class PeerExchange:
    """Peer-mapped workspace of one rank for the CFG x SP step.

    arena (sp group):   qkv  bf16 [3, Hg, S, 64]   my head group over the WHOLE sequence, filled by every sp rank's QKV epilogue
                        cat  bf16 [S/sp, ldc]      [attention out | MLP hidden] of my token chunk; the attention columns are
                                                   filled by every sp rank's attention epilogue
                        flags uint32 [8]           barrier slots
    world arena:        vel  [cfg_ways, ...]       the two branches' velocities, published to every rank by pf_peer_bcast
                        head fp32 [n_last, 64]     (sp > 1) output-head rows, published inside the sp group
                        flags uint32 [8]
    Sized once for the largest sequence (`max_seq`); a new (seq, widths) layout only re-slices the arena."""

    def __init__(self, lay: ParallelLayout, max_seq: int, hp: int, ldc: int, head_cols: int, max_last: int, vel_bytes: int):
        assert dist.is_initialized()
        self.lay = lay
        sp = lay.sp
        hg = hp // sp
        world = lay.world
        rank = lay.rank
        sp_ranks = [lay.cfg_rank * sp + i for i in range(sp)]
        a256 = lambda n: (n + 255) // 256 * 256
        self.off_flags = 0
        self.off_qkv = 256
        self.off_cat = self.off_qkv + a256(3 * hg * max_seq * 64 * 2)
        sl_max = (max_seq + sp - 1) // sp
        self.off_head = self.off_cat + a256(sl_max * ldc * 2)
        self.sp_bytes = self.off_head + a256(max_last * head_cols * 4)
        self.max_seq, self.hg, self.ldc, self.head_cols, self.max_last = max_seq, hg, ldc, head_cols, max_last
        self.sp_buf = PeerBuffer(self.sp_bytes, sp_ranks, rank)
        self.w_off_flags = 0
        self.w_off_vel = 256
        self.vel_bytes = a256(vel_bytes)
        self.world_buf = PeerBuffer(self.w_off_vel + lay.cfg_ways * self.vel_bytes, list(range(world)), rank)
        self.epoch_sp = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.epoch_world = torch.zeros(1, dtype=torch.int32, device="cuda")
        self._g_sp_flags = self.sp_buf.group(self.off_flags)
        self._g_world_flags = self.world_buf.group(self.w_off_flags)
        torch.cuda.synchronize()
        dist.barrier()

    def close(self) -> None:
        self.sp_buf.close()
        self.world_buf.close()

    # -- views of the local arena ------------------------------------------------------------------------------------
    def qkv(self, seq: int) -> torch.Tensor:
        return self.sp_buf.view(self.off_qkv, (3, self.hg, seq, 64), torch.bfloat16)

    def cat(self, sl: int) -> torch.Tensor:
        return self.sp_buf.view(self.off_cat, (1, sl, self.ldc), torch.bfloat16)

    def head(self, n_last: int) -> torch.Tensor:
        return self.sp_buf.view(self.off_head, (1, n_last, self.head_cols), torch.float32)

    def vel(self, shape, dtype) -> torch.Tensor:
        n = 1
        for s in shape[1:]:
            n *= int(s)
        es = torch.empty(0, dtype=dtype).element_size()
        assert n * es <= self.vel_bytes
        # branches are vel_bytes apart; expose [cfg_ways, ...] through a strided view
        flat = self.world_buf.local[self.w_off_vel:self.w_off_vel + self.lay.cfg_ways * self.vel_bytes]
        return flat.view(self.lay.cfg_ways, self.vel_bytes)[:, :n * es].view(dtype).view(self.lay.cfg_ways, *shape[1:])

    # -- collective pieces ---------------------------------------------------------------------------------------------
    def barrier_sp(self) -> None:
        from . import _lib
        import ctypes as C
        _lib.check(_lib.load().pf_peer_barrier(C.byref(self._g_sp_flags), self.epoch_sp.data_ptr(), _lib.stream_ptr()),
                   "pf_peer_barrier(sp)")

    def barrier_world(self) -> None:
        from . import _lib
        import ctypes as C
        _lib.check(_lib.load().pf_peer_barrier(C.byref(self._g_world_flags), self.epoch_world.data_ptr(), _lib.stream_ptr()),
                   "pf_peer_barrier(world)")

    def bcast(self, buf: PeerBuffer, src: torch.Tensor, dst_offset: int) -> None:
        from . import _lib
        import ctypes as C
        g = buf.group(0)
        nb = src.numel() * src.element_size()
        assert src.is_contiguous() and nb % 16 == 0 and dst_offset % 16 == 0
        _lib.check(_lib.load().pf_peer_bcast(C.byref(g), src.data_ptr(), nb, dst_offset, _lib.stream_ptr()), "pf_peer_bcast")


def ensure_peer_exchange(owner, lay: ParallelLayout, seq: int, last_tokens: int, hp: int, ldc: int, head_cols: int,
                         vel_bytes: int) -> PeerExchange:
    """The peer arena of `owner` (a B200FluxTransformer / B200MMDiT), (re)built collectively when a call needs more room than
    it has.  Every rank sees the same shapes, so every rank takes the same decision.  `owner.peer_max_seq / peer_max_last /
    peer_max_vel_bytes` pre-size it (one allocation for a whole sampler run)."""
    px = getattr(owner, "_px", None)
    if (px is None or seq > px.max_seq or last_tokens > px.max_last or vel_bytes > px.vel_bytes or px.ldc != ldc
            or px.head_cols != head_cols):
        if px is not None:
            torch.cuda.synchronize()
            dist.barrier()
            if hasattr(owner, "_graphs"):
                owner._graphs.clear()           # captured launches point into the old arena
            px.close()
        px = PeerExchange(lay, max(seq, getattr(owner, "peer_max_seq", 0)), hp, ldc, head_cols,
                          max(last_tokens, getattr(owner, "peer_max_last", 0)),
                          max(vel_bytes, getattr(owner, "peer_max_vel_bytes", 0)))
        owner._px = px
    return px
