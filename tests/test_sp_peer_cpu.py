"""Host-side refusals of the sequence-parallel peer-store paths (pf_gemm_desc.peer_*, pf_attn_desc.peer_*, pf_peer_barrier,
pf_peer_bcast), and the peer-store arguments the step builds (sp.peer_store_args).  Validation happens before any CUDA call;
pointers are dummies, never dereferenced, so nothing here needs a GPU."""
import ctypes as C

import pytest

from pyramid_flow_b200 import _lib
from pyramid_flow_b200 import sp as SP
from pyramid_flow_b200._lib import AttnDesc, GemmDesc, PeerGroup, PF_EPI_QKV_ROPE, PF_EPI_STORE_BF16

DUMMY = 0x10000


def _err():
    return _lib.load().pf_last_error().decode()


def _qkv_desc(heads=4, sp=2, seq=512, row_begin=0, rows=256, row0=0):
    """A QKV_ROPE launch of one rank's chunk with peer stores that passes validation (up to the first CUDA call)."""
    d = GemmDesc()
    d.a, d.lda, d.w, d.k = DUMMY, 256, DUMMY, 256
    d.batches, d.rows_per_batch, d.row_begin, d.row_count = 1, rows, row_begin, rows - row_begin
    d.n, d.epilogue = 3 * heads * 64, PF_EPI_QKV_ROPE
    d.q_out = d.k_out = d.v_out = d.q_norm_w = d.k_norm_w = DUMMY
    d.heads, d.head_dim, d.seq_len = heads, 64, rows
    d.out_row_begin = row_begin
    d.peer_count, d.peer_heads, d.peer_seq, d.peer_row0 = sp, SP.padded_heads(heads, sp) // sp, seq, row0
    for i in range(sp):
        d.peer_qkv[i] = DUMMY + 0x100000 * i
    return d


def _attn_desc(heads=2, sp=2, seq=512, ldo=None, col_begin=128):
    d = AttnDesc()
    d.q = d.k = d.v = d.seg = d.time = d.tile_sched = DUMMY
    d.batch, d.heads, d.seq, d.head_dim, d.scale = 1, heads, seq, 64, 0.125
    d.sched_stride = 1 + (seq + 127) // 128
    d.ldo = ldo if ldo is not None else sp * heads * 64 + 256
    d.peer_count, d.peer_chunk_rows, d.peer_col_begin = sp, seq // sp, col_begin
    for i in range(sp):
        d.peer_out[i] = DUMMY + 0x100000 * i
    return d


def _gemm_refused(d, *words):
    rc = _lib.load().pf_gemm_bf16(C.byref(d), None)
    msg = _err()
    assert rc < 0 and all(w in msg for w in words), (rc, msg)


def _attn_refused(d, *words):
    rc = _lib.load().pf_attn_fwd_masked(C.byref(d), None)
    msg = _err()
    assert rc < 0 and all(w in msg for w in words), (rc, msg)


def test_gemm_peer_refusals():
    d = _qkv_desc()
    d.epilogue, d.out, d.ldo = PF_EPI_STORE_BF16, DUMMY, 3 * 4 * 64
    _gemm_refused(d, "QKV_ROPE")
    d = _qkv_desc()
    d.batches = 2
    _gemm_refused(d, "batches == 1")
    d = _qkv_desc(heads=30, sp=4)
    d.peer_heads = 7                                     # 7 x 4 = 28 < 30 heads: heads 28, 29 would have no owner
    _gemm_refused(d, "bad peer layout")
    d = _qkv_desc(seq=512, row_begin=10, rows=256, row0=256)
    d.peer_row0 = 257                                    # 257 + 10 + 246 = 513 > 512
    _gemm_refused(d, "bad peer layout")
    d = _qkv_desc(seq=512, row_begin=10, rows=256, row0=256)
    d.peer_row0 = -1
    _gemm_refused(d, "bad peer layout")
    d = _qkv_desc(sp=4)
    d.peer_qkv[3] = None
    _gemm_refused(d, "peer_qkv[3] is null")
    d = _qkv_desc(sp=8)
    d.peer_count = 9
    _gemm_refused(d, "bad peer layout")
    for off in (2, 8):                                   # the staged epilogue stores 16-byte vectors
        d = _qkv_desc(sp=4)
        d.peer_qkv[2] = DUMMY + 0x200000 + off
        _gemm_refused(d, "peer_qkv[2]", "16-byte aligned")


def test_attn_peer_refusals():
    d = _attn_desc()
    d.batch = 2
    _attn_refused(d, "bad peer layout")
    d = _attn_desc(sp=4, seq=600)
    d.peer_chunk_rows = 149                              # 4 x 149 = 596 < 600: the last rows would have no owner
    _attn_refused(d, "bad peer layout")
    d = _attn_desc(col_begin=132)
    _attn_refused(d, "bad peer layout")
    d = _attn_desc(sp=4)
    d.peer_out[1] = None
    _attn_refused(d, "peer_out[1] is null")


def test_attn_peer_columns_must_fit_the_row():
    """A rank's head group [peer_col_begin, peer_col_begin + heads*64) must end inside the row; past ldo the stores would
    run into the next row's MLP columns."""
    heads, sp = 8, 4
    ldc = sp * heads * 64 + 4 * 512                      # [attention out of every head group | MLP hidden]
    last = (sp - 1) * heads * 64
    _lib.load()
    d = _attn_desc(heads=heads, sp=sp, ldo=ldc, col_begin=ldc - heads * 64 + 8)
    _attn_refused(d, "exceed the row stride")
    d = _attn_desc(heads=heads, sp=sp, ldo=last + heads * 64 - 8, col_begin=last)
    _attn_refused(d, "exceed the row stride")
    d = _attn_desc(heads=heads, sp=sp, ldo=ldc, col_begin=-8)
    _attn_refused(d, "exceed the row stride")


@pytest.mark.parametrize("off", [2, 8])
def test_attn_peer_out_must_be_16_byte_aligned(off):
    d = _attn_desc(sp=4)
    d.peer_out[3] = DUMMY + 0x300000 + off
    _attn_refused(d, "peer_out[3]", "16-byte aligned")


def _group(n, my_index=0):
    g = PeerGroup()
    for i in range(min(n, 8)):
        g.ptr[i] = DUMMY + 0x1000 * i
    g.n, g.my_index = n, my_index
    return g


def test_barrier_refusals():
    lib = _lib.load()
    for n, me in ((0, 0), (9, 0), (4, 4), (4, -1), (1, 1)):
        g = _group(n, me)
        assert lib.pf_peer_barrier(C.byref(g), DUMMY, None) < 0 and "bad group" in _err(), (n, me)
    assert lib.pf_peer_barrier(C.byref(_group(2)), None, None) < 0 and "bad group" in _err()
    assert lib.pf_peer_barrier(None, DUMMY, None) < 0 and "bad group" in _err()


def test_bcast_refusals():
    lib = _lib.load()
    for n in (0, 9):
        assert lib.pf_peer_bcast(C.byref(_group(n)), DUMMY, 64, 0, None) < 0 and "bad group" in _err(), n
    g = _group(4, 2)
    for src, nbytes, off in ((DUMMY, 24, 0), (DUMMY, 0, 0), (DUMMY, -16, 0), (DUMMY, 64, 8), (DUMMY + 8, 64, 0),
                             (DUMMY + 4, 64, 16)):
        assert lib.pf_peer_bcast(C.byref(g), src, nbytes, off, None) < 0 and "16 bytes" in _err(), (src, nbytes, off)
    assert lib.pf_peer_bcast(C.byref(g), None, 64, 0, None) < 0 and "bad group" in _err()


@pytest.mark.parametrize("heads,sp,seq", [(30, 2, 600), (30, 4, 600), (30, 8, 600), (24, 4, 600), (4, 2, 600),
                                          (30, 4, 15488), (30, 8, 15488)])
def test_peer_store_args_cover_every_row_and_head_once(heads, sp, seq):
    """The descriptors of the sp ranks, taken together, send every (head, token) of the QKV epilogue to exactly one gathered
    row, and every (token, head group) of the attention epilogue to exactly one `cat` row and column block."""
    hp = SP.padded_heads(heads, sp)
    qkv_ptrs = [0x100000 * (i + 1) for i in range(sp)]
    cat_ptrs = [0x900000 * (i + 1) for i in range(sp)]
    seen_qkv, seen_cat = set(), set()
    for r in range(sp):
        pq, po = SP.peer_store_args(seq, sp, r, hp, qkv_ptrs, cat_ptrs)
        c0, c1 = SP.chunk_bounds(seq, sp, r)
        assert pq["peer_ptrs"] == qkv_ptrs and po["peer_ptrs"] == cat_ptrs
        assert pq["peer_heads"] * sp == hp and pq["peer_seq"] == seq
        assert po["peer_chunk_rows"] * sp == seq and po["peer_col_begin"] % 8 == 0
        # the kernels' index arithmetic (pf_gemm.cu qkv epilogues, pf_attn.cu epilogue) on this rank's descriptors
        for h in range(heads):
            owner, hl = h // pq["peer_heads"], h % pq["peer_heads"]
            for pos in range(c1 - c0):
                seen_qkv.add((owner, hl, pq["peer_row0"] + pos))
        for hl in range(hp // sp):
            for q in range(seq):
                owner = q // po["peer_chunk_rows"]
                seen_cat.add((owner, q - owner * po["peer_chunk_rows"], po["peer_col_begin"] + hl * 64))
    hg = hp // sp
    assert len(seen_qkv) == heads * seq
    assert seen_qkv == {(h // hg, h % hg, p) for h in range(heads) for p in range(seq)}
    assert len(seen_cat) == seq * hp
    assert seen_cat == {(q // (seq // sp), q % (seq // sp), h * 64) for h in range(hp) for q in range(seq)}
