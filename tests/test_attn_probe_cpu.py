"""The attention probe harness (tests/attn_probe.py) on the CPU: with a float64 attention standing in for the kernels, the
probe construction and the checks must pass; a planted zero block and a leaked element must both be named; the schedule
mutations of the sensitivity tests must change exactly one block and stay in bounds."""
import torch

from oracle import flux_oracle as FO
from pyramid_flow_b200 import ops
from pyramid_flow_b200.dit import build_seq_plan
from tests import attn_probe as AP


def _fake_fwd(q, k, v, allowed, scale):
    """fp64 masked attention, output rounded to bf16 as the kernel stores it: [B, S, H * 64]."""
    s = (q.double() @ k.double().transpose(-1, -2)) * scale
    p = torch.softmax(s.masked_fill(~allowed[:, None], float("-inf")), dim=-1)
    return AP.head_columns((p @ v.double()).bfloat16())


def _fake_bwd(q, k, v, out, dout, allowed, scale):
    """fp64 gradients on the kernel's contract (delta = rowsum(dO o out) of the stored bf16 out), rounded to bf16:
    (dq, dk, dv) [B, H, S, 64]."""
    b, h, n, _ = q.shape
    qq, kk, vv = (t.double() for t in (q, k, v))
    o, do = (t.double().view(b, n, h, 64).transpose(1, 2) for t in (out, dout))
    s = (qq @ kk.transpose(-1, -2)) * scale
    p = torch.softmax(s.masked_fill(~allowed[:, None], float("-inf")), dim=-1)
    ds = p * (do @ vv.transpose(-1, -2) - (do * o).sum(-1, keepdim=True))
    return tuple(t.bfloat16() for t in (scale * ds @ kk, scale * ds.transpose(-1, -2) @ qq, p.transpose(-1, -2) @ do))


def _pyramid_plan():
    shapes = [(2, 16, 2, 12, 20), (2, 16, 1, 24, 40), (2, 16, 1, 48, 80)]
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[0, 37:] = 0
    plan = build_seq_plan(shapes, mask, (16, 24, 24), 2, "cpu")
    allowed = FO.attention_mask(FO.token_segments(mask, plan.video_len), FO.sequence_ids(shapes, 128)[:, 0])[:, 0]
    return plan, allowed


def test_probe_identities_hold_on_an_fp64_attention():
    g = torch.Generator().manual_seed(0)
    seg, time = AP.restated_layout(2, 24, [(6, 40)])
    allowed = AP.dense_mask(seg, time)
    b, s = seg.shape
    h = AP.heads_for(s)
    q, k = AP.random_heads(b, s, h, g, "cpu"), AP.random_heads(b, s, h, g, "cpu")
    v = AP.identity_heads(b, s, h, "cpu")
    out = _fake_fwd(q, k, v, allowed, AP.SCALE)
    p_ref, _ = AP.fwd_reference(q, k, allowed, AP.SCALE)
    rep = AP.check_probs("fwd", out, p_ref, allowed, AP.rel_bound_fwd(AP.SCALE, AP.norm_product_max(q, k)))
    assert rep.ok(), str(rep)
    assert 2.0 ** -10 < rep.worst <= 2.0 ** -8, rep.worst          # one bf16 rounding of P: the probe reads P itself
    assert bool((out[..., s:] == 0).all()) and out.shape[-1] > s

    # the three backward probes, each with fp64 gradients of the same bf16 inputs standing in for the kernel
    eye_do = AP.head_columns(AP.identity_heads(b, s, h, "cpu"))
    dout = AP.head_columns(AP.random_heads(b, s, h, g, "cpu"))
    for probe in ("dv", "dq", "dk"):
        qq = AP.identity_heads(b, s, h, "cpu") if probe == "dk" else q
        kk = AP.identity_heads(b, s, h, "cpu") if probe == "dq" else k
        vv = AP.random_heads(b, s, h, g, "cpu")
        do = eye_do if probe == "dv" else dout
        o = _fake_fwd(qq, kk, vv, allowed, AP.SCALE)
        dq, dk, dv = _fake_bwd(qq, kk, vv, o, do, allowed, AP.SCALE)
        ref = AP.bwd_reference(qq, kk, vv, o, do, allowed, AP.SCALE)
        if probe == "dv":
            rep = AP.check_probs("dv", AP.head_columns(dv), ref.pt, allowed.transpose(1, 2), ref.rel_dv)
        elif probe == "dq":
            rep = AP.check_grads("dq", AP.head_columns(dq) / AP.SCALE, ref.ds, ref.ds_bound, allowed)
        else:
            rep = AP.check_grads("dk", AP.head_columns(dk) / AP.SCALE, ref.dst, ref.dst_bound, allowed.transpose(1, 2))
        assert rep.ok(), str(rep)
        assert rep.worst > 0


def test_checks_name_a_zeroed_block_and_a_leaked_element():
    plan, allowed = _pyramid_plan()
    b, s = plan.seg.shape
    h = AP.heads_for(s)
    g = torch.Generator().manual_seed(1)
    q, k = AP.random_heads(b, s, h, g, "cpu"), AP.random_heads(b, s, h, g, "cpu")
    out = _fake_fwd(q, k, AP.identity_heads(b, s, h, "cpu"), allowed, AP.SCALE)
    p_ref, _ = AP.fwd_reference(q, k, allowed, AP.SCALE)
    bound = AP.rel_bound_fwd(AP.SCALE, AP.norm_product_max(q, k))
    assert AP.check_probs("clean", out, p_ref, allowed, bound).ok()

    bad = out.clone()
    block = AP.tile_region(bad.shape, 1, 9, 3)          # video rows of sample 1 against a fully allowed kv tile
    assert bool(allowed[1, 9 * 128:10 * 128, 3 * 128:4 * 128].all())
    bad[block] = 0
    leak = (0, 1000, 100)                               # a video query and a padded text key of sample 0
    assert not bool(allowed[leak])
    bad[leak] = 1e-3
    rep = AP.check_probs("planted", bad, p_ref, allowed, bound)
    assert not rep.ok()
    assert torch.equal(rep.missing, block & AP.pad_cols(allowed, bad.shape[-1], False))
    assert rep.leaked.nonzero().tolist() == [list(leak)]
    assert not bool((rep.inexact & ~block).any())
    text = str(rep)
    assert "missing: 16384 elements" in text and "rows 1152..1279, cols 384..511" in text
    assert "leaked: 1 elements" in text and str(leak) in text

    # the dS check: a planted zero block is missing wherever |dS| clears the bound, and a wrong sign is named too
    ds = torch.randn(1, 256, 256, dtype=torch.float64)
    ok = torch.ones(1, 256, 256, dtype=torch.bool)
    bnd = 2.0 ** -8 * ds.abs() + 1e-6
    got = ds.bfloat16().clone()
    got[0, 128:, :128] = 0
    got[0, 3, 200] = -got[0, 3, 200]
    rep = AP.check_grads("planted ds", got, ds, bnd, ok)
    zero = AP.tile_region(got.shape, 0, 1, 0)
    want = (zero & (ds.abs() > bnd))
    want[0, 3, 200] = bool(ds[0, 3, 200].abs() > bnd[0, 3, 200])
    assert torch.equal(rep.missing, want) and not bool(rep.leaked.any())


def test_schedule_mutations_change_exactly_one_block():
    plan, allowed = _pyramid_plan()
    sched = plan.sched.cpu()
    b, tiles, stride = sched.shape
    before = AP.sched_entries(sched)
    for bi in range(b):
        for t in range(tiles):
            n = int(sched[bi, t, 0])
            for i in range(n):
                e = int(sched[bi, t, 1 + i])
                dropped = AP.drop_entry(sched, bi, t, i)
                assert AP.sched_entries(dropped) == before - {(bi, t, e >> 1, e & 1)}
                assert int(dropped[bi, t, 0]) == n - 1 and bool((dropped[bi, t, n:] == 0).all())
                assert torch.equal(dropped[bi, t, 1:n], torch.cat([sched[bi, t, 1:1 + i], sched[bi, t, 2 + i:1 + n]]))
                others = torch.ones(b, tiles, dtype=torch.bool)
                others[bi, t] = False
                assert torch.equal(dropped[others], sched[others])
                if e & 1:
                    cleared = AP.clear_partial(sched, bi, t, i)
                    assert AP.sched_entries(cleared) ^ before == {(bi, t, e >> 1, 1), (bi, t, e >> 1, 0)}
                    assert int((cleared != sched).sum()) == 1
                for m in [dropped] + ([cleared] if e & 1 else []):
                    ks = [x[2] for x in AP.sched_entries(m)]
                    assert min(ks) >= 0 and max(ks) < tiles
                    assert bool((m[..., 0] <= tiles).all())
    # the kv-major transpose builds from a mutated q schedule and differs from the plan's by the same one block
    kv = ops.attn_build_kv_schedule(sched, plan.seq)
    e = int(sched[1, 9, 2])
    kv_dropped = ops.attn_build_kv_schedule(AP.drop_entry(sched, 1, 9, 1), plan.seq)
    assert AP.sched_entries(kv) - AP.sched_entries(kv_dropped) == {(1, e >> 1, 9, e & 1)}
    assert AP.sched_entries(kv_dropped) <= AP.sched_entries(kv)
    # the probe's layout really is the reference mask: every allowed pair lies in a scheduled tile
    assert plan.allowed_pairs == int(allowed.sum())
