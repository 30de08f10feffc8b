"""Host-side logic of the drop-in (no GPU): sequence plan vs the oracle's restatement of merge_input, C-ABI exports."""
import ctypes as C
import re
from pathlib import Path

import torch

from oracle import flux_oracle as FO
from pyramid_flow_b200 import _lib, ops
from pyramid_flow_b200.dit import build_position_ids, build_rope_table, build_seq_plan

ROOT = Path(__file__).resolve().parent.parent


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    header = (ROOT / "include" / "pf_b200.h").read_text()
    declared = set(re.findall(r"PF_API\s+[\w\s\*]+?\b(pf_\w+)\s*\(", header))
    assert declared, "no PF_API declarations parsed"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    for s in declared:
        assert hasattr(lib, s), s
    assert lib.pf_version() >= 100


def test_no_cpu_fallback_without_gpu():
    if torch.cuda.is_available():
        return
    lib = _lib.load()
    assert lib.pf_device_check() != 0
    try:
        _lib.require_device()
    except RuntimeError as e:
        assert "pf_device_check" in str(e)
    else:
        raise AssertionError("require_device must fail loudly without a GPU")


def test_ids_and_rope_match_oracle():
    shapes = [(2, 16, 3, 12, 20), (2, 16, 1, 24, 40), (2, 16, 1, 48, 80)]
    ids_o = FO.sequence_ids(shapes, 128)
    thw = [(s[2], s[3] // 2, s[4] // 2) for s in shapes]
    ids = build_position_ids(thw, 128)
    assert torch.equal(ids, ids_o)
    # coarser clips sit at fractional positions of the finest grid (0.5, 2.5, ... at half resolution)
    half = ids[128 + 3 * 6 * 10: 128 + 3 * 6 * 10 + 12 * 20].reshape(12, 20, 3)
    assert half[0, 0, 1].item() == 0.5 and half[1, 0, 1].item() == 2.5 and half[0, 1, 2].item() == 2.5
    assert torch.equal(build_rope_table(ids, (16, 24, 24)), FO.rope_table(ids_o, (16, 24, 24)))


def test_plan_schedule_covers_exactly_the_allowed_pairs():
    shapes = [(2, 16, 2, 12, 20), (2, 16, 1, 24, 40), (2, 16, 1, 48, 80)]
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[0, 37:] = 0
    plan = build_seq_plan(shapes, mask, (16, 24, 24), 2, "cpu")
    seg_o = FO.token_segments(mask, plan.video_len)
    ids_o = FO.sequence_ids(shapes, 128)
    dense = FO.attention_mask(seg_o, ids_o[:, 0])[:, 0]
    assert plan.allowed_pairs == int(dense.sum())
    assert torch.equal(plan.seg.long(), seg_o)
    # every allowed pair lies in a scheduled tile; every unflagged tile is fully allowed
    b, s = plan.seg.shape
    qt_n = (s + 127) // 128
    for bi in range(b):
        covered = torch.zeros(s, s, dtype=torch.bool)
        for qt in range(qt_n):
            row = plan.sched[bi, qt]
            for e in row[1:1 + int(row[0])].tolist():
                kt, flag = e >> 1, e & 1
                q0, q1, k0, k1 = qt * 128, min(s, qt * 128 + 128), kt * 128, min(s, kt * 128 + 128)
                covered[q0:q1, k0:k1] = True
                if not flag:
                    assert bool(dense[bi, q0:q1, k0:k1].all())
        assert not bool((dense[bi] & ~covered).any())


def test_vae_context_parallel_schedule():
    """cp_frame_split: rounds cover the clip in time order; round 0 / rank 0 holds the image frame; only the last round is
    partial; every share that has a successor owns >= 2 frames (its halo source is its own data)."""
    from pyramid_flow_b200.vae import B200CausalVAE as V
    for n in (5, 9, 12, 17, 31, 64):
        for world in (2, 4, 8):
            for c in (2, 4):
                rounds = V.cp_frame_split(n, world, c)
                flat = [x for r in rounds for x in r]
                assert flat[0][0] == 0 and flat[-1][1] == n
                assert all(flat[i][1] == flat[i + 1][0] for i in range(len(flat) - 1))
                assert rounds[0][0] == (0, min(n, c + 1))
                for k, ranges in enumerate(rounds):
                    assert len(ranges) == world
                    for r, (a, b) in enumerate(ranges):
                        full = c + (1 if (k == 0 and r == 0) else 0)
                        assert b - a <= full
                        has_successor = (r + 1 < world and ranges[r + 1][1] > ranges[r + 1][0]) or (r == world - 1 and k + 1 < len(rounds))
                        if has_successor:
                            assert b - a == full >= 2


def test_c_abi_rejects_bad_arguments_with_a_message():
    """Error behaviour of the C-ABI (INTEGRATION.md: int status + pf_last_error): argument validation is host-side and happens
    before any CUDA call, so it is checkable without a GPU.  Pointers are dummies — they are never dereferenced here."""
    from pyramid_flow_b200._lib import AttnDesc, ConvDesc, GemmDesc
    lib = _lib.load()
    dummy = 0x1000

    def err():
        return lib.pf_last_error().decode()

    a = AttnDesc()
    a.q = a.k = a.v = a.out = a.seg = a.time = a.tile_sched = dummy
    a.batch, a.heads, a.seq, a.head_dim, a.ldo, a.sched_stride = 1, 2, 256, 32, 128, 3
    assert lib.pf_attn_fwd_masked(C.byref(a), None) < 0 and "head_dim" in err()
    a.head_dim, a.sched_stride = 64, 1
    assert lib.pf_attn_fwd_masked(C.byref(a), None) < 0 and "stride" in err()
    a.sched_stride, a.q_row_begin = 3, 100
    assert lib.pf_attn_fwd_masked(C.byref(a), None) < 0 and "q_row_begin" in err()
    assert lib.pf_attn_fwd_masked(None, None) < 0 and "null" in err()

    c = ConvDesc()
    c.x = c.wgt = c.out = dummy
    c.b, c.t, c.h, c.w, c.cin, c.cout, c.kt, c.kh, c.kw = 1, 1, 8, 8, 10, 64, 3, 3, 3
    c.store_channels, c.out_c = 64, 64
    assert lib.pf_causal_conv3d(C.byref(c), None) < 0 and "cin" in err()
    c.cin, c.kt = 64, 2
    assert lib.pf_causal_conv3d(C.byref(c), None) < 0 and "kernel" in err()
    c.kt, c.stride_h, c.stride_w = 3, 2, 1
    assert lib.pf_causal_conv3d(C.byref(c), None) < 0 and "stride" in err()
    c.stride_w, c.store_mode, c.out_c = 2, 1, 16
    assert lib.pf_causal_conv3d(C.byref(c), None) < 0      # strided convs are plain-store only

    g = GemmDesc()
    g.a = g.w = g.out = dummy
    g.batches, g.rows_per_batch, g.row_count, g.n, g.k, g.lda, g.ldo = 1, 128, 128, 64, 64, 64, 64
    g.epilogue = 17
    assert lib.pf_gemm_bf16(C.byref(g), None) < 0 and "epilogue" in err()


def test_pair_schedule_is_the_union_of_the_two_tile_rows():
    """pf_attn_build_pair_schedule (host code): pair p = q tiles (q_tiles-2-2p, q_tiles-1-2p);
    its row is the sorted union of the two tiles' kv lists; per-tile flags reproduce each tile's own list and mask bits; a
    missing lower tile (odd q_tiles) contributes nothing."""
    import torch
    from pyramid_flow_b200 import ops
    g = torch.Generator().manual_seed(0)
    for seq, lens in [(77, [77]), (128 + 60 * 5, [128 + 60] + [60] * 4), (128 + 200 + 1000 + 1700, [328, 1000, 1700]),
                      (77 + 240 * 9 + 13, [77 + 240] + [240] * 8 + [13])]:
        tim = torch.cat([torch.full((n,), i) for i, n in enumerate(lens)]).int()[None].repeat(2, 1)
        seg = torch.ones(2, seq, dtype=torch.int32)
        seg[1, 10:int(torch.randint(20, 60, (1,), generator=g))] = 0
        sched, pairs = ops.attn_build_schedule(seg, tim)
        pso = ops.attn_build_pair_schedule(sched, seq, seg, tim)
        ps = pso.sched
        qt = (seq + 127) // 128
        assert ps.shape == (2, (qt + 1) // 2, sched.shape[-1])
        for b in range(2):
            for p in range((qt + 1) // 2):
                hi, lo = qt - 1 - 2 * p, qt - 2 - 2 * p
                n = int(ps[b, p, 0])
                ent = ps[b, p, 1:1 + n].tolist()
                kts = [e >> 4 for e in ent]
                assert kts == sorted(set(kts)), "union must be strictly increasing"
                assert all((e & 0xF) != 0 for e in ent), "every entry is needed by at least one tile"
                for x, t in ((0, lo), (1, hi)):
                    own = [((e >> 4) << 1) | (((e >> (2 * x)) & 2) >> 1) for e in ent if (e >> (2 * x)) & 1]
                    want = [] if t < 0 else sched[b, t, 1:1 + int(sched[b, t, 0])].tolist()
                    assert own == want, (seq, b, p, x)
                assert bool((ps[b, p, 1 + n:] == 0).all())
                # row masks of the partial tiles == the dense mask definition (F:318-350), bit i of word w = kv column 32 w + i
                for e_i, e in enumerate(ent):
                    for x, t in ((0, lo), (1, hi)):
                        blk = int(pso.mask_index[b, p, 2 * e_i + x])
                        if ((e >> (2 * x)) & 3) != 3:
                            assert blk == -1
                            continue
                        words = pso.mask_bits[blk].to(torch.int64) & 0xFFFFFFFF            # [128, 4]
                        bits = ((words[:, :, None] >> torch.arange(32)[None, None, :]) & 1).reshape(128, 128).bool()
                        q = torch.arange(t * 128, t * 128 + 128)
                        kv = torch.arange((e >> 4) * 128, (e >> 4) * 128 + 128)
                        qv, kvv = q < seq, kv < seq
                        qc, kc = q.clamp(max=seq - 1), kv.clamp(max=seq - 1)
                        dense = (seg[b][qc][:, None] == seg[b][kc][None, :]) & (tim[b][qc][:, None] >= tim[b][kc][None, :])
                        dense &= qv[:, None] & kvv[None, :]
                        assert torch.equal(bits, dense), (seq, b, p, e_i, x)


def test_group_schedule_is_the_union_of_the_three_tile_rows():
    """pf_attn_build_group_schedule / _masks (host code): group g = q tiles
    q_tiles-3-3g .. q_tiles-1-3g; its row is the sorted union of the tiles' kv lists, per-tile flags reproduce each tile's own
    list, missing leading tiles contribute nothing, and the row masks equal the dense mask definition (F:318-350)."""
    import torch
    from pyramid_flow_b200 import ops
    g_ = torch.Generator().manual_seed(1)
    for seq, lens in [(77, [77]), (128 + 60 * 5, [128 + 60] + [60] * 4), (128 + 200 + 1000 + 1700, [328, 1000, 1700]),
                      (77 + 240 * 9 + 13, [77 + 240] + [240] * 8 + [13])]:
        tim = torch.cat([torch.full((n,), i) for i, n in enumerate(lens)]).int()[None].repeat(2, 1)
        seg = torch.ones(2, seq, dtype=torch.int32)
        seg[1, 10:int(torch.randint(20, 60, (1,), generator=g_))] = 0
        sched, pairs = ops.attn_build_schedule(seg, tim)
        pso = ops.attn_build_pair_schedule(sched, seq, seg, tim)
        assert pso.group3.mask_bits is pso.mask_bits, "the plan's group schedule indexes the pair schedule's block pool"
        qt = (seq + 127) // 128
        n_groups = (qt + 2) // 3
        # both forms: standalone (own block pool) and the one every plan carries (blocks shared with the pair schedule)
        for gs in (ops.attn_build_group_schedule(sched, seq, seg, tim, 3), pso.group3):
          assert gs.sched.shape == (2, n_groups, sched.shape[-1]) and gs.mask_index.shape == (2, n_groups, 3 * sched.shape[-1])
          for b in range(2):
              for gi in range(n_groups):
                  top = qt - 1 - 3 * gi
                  n = int(gs.sched[b, gi, 0])
                  ent = gs.sched[b, gi, 1:1 + n].tolist()
                  kts = [e >> 8 for e in ent]
                  assert kts == sorted(set(kts)), "union must be strictly increasing"
                  assert all((e & 0x3F) != 0 for e in ent), "every entry is needed by at least one tile"
                  assert bool((gs.sched[b, gi, 1 + n:] == 0).all())
                  for x in range(3):
                      t = top - (2 - x)
                      own = [((e >> 8) << 1) | (((e >> (2 * x)) & 2) >> 1) for e in ent if (e >> (2 * x)) & 1]
                      want = [] if t < 0 else sched[b, t, 1:1 + int(sched[b, t, 0])].tolist()
                      assert own == want, (seq, b, gi, x)
                      for e_i, e in enumerate(ent):
                          blk = int(gs.mask_index[b, gi, 3 * e_i + x])
                          if ((e >> (2 * x)) & 3) != 3:
                              assert blk == -1
                              continue
                          words = gs.mask_bits[blk].to(torch.int64) & 0xFFFFFFFF            # [128, 4]
                          bits = ((words[:, :, None] >> torch.arange(32)[None, None, :]) & 1).reshape(128, 128).bool()
                          q = torch.arange(t * 128, t * 128 + 128)
                          kv = torch.arange((e >> 8) * 128, (e >> 8) * 128 + 128)
                          qv, kvv = q < seq, kv < seq
                          qc, kc = q.clamp(max=seq - 1), kv.clamp(max=seq - 1)
                          dense = (seg[b][qc][:, None] == seg[b][kc][None, :]) & (tim[b][qc][:, None] >= tim[b][kc][None, :])
                          dense &= qv[:, None] & kvv[None, :]
                          assert torch.equal(bits, dense), (seq, b, gi, e_i, x)
