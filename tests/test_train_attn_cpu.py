"""Host-side logic of the trainable masked attention (no GPU): the kv-major schedule, the seg / time ids the merge_input
wrapper derives, and the argument checks of the C entries."""
import ctypes as C

import pytest
import torch

from pyramid_flow_b200 import _lib, ops, training


def _dense(seg, time):
    return (seg[:, :, None] == seg[:, None, :]) & (time[:, :, None] >= time[:, None, :])


def _pyramid_layout(g, batch, text, clips):
    """seg / time [batch, S] of one stage: `text` text tokens (randomly padded per sample, seg 0), then the clips'
    tokens (t_i frames of n_i tokens each, consecutive time stamps from 0)."""
    segs, times = [], []
    for _ in range(batch):
        valid = int(torch.randint(1, text + 1, (1,), generator=g))
        seg = [1] * valid + [0] * (text - valid)
        time = [0] * text
        stamp = 0
        for t, n in clips:
            for f in range(t):
                seg += [1] * n
                time += [stamp + f] * n
            stamp += t
        segs.append(seg)
        times.append(time)
    return torch.tensor(segs, dtype=torch.int32), torch.tensor(times, dtype=torch.int32)


LAYOUTS = [
    (77, [(1, 60)]),
    (128, [(2, 40), (1, 160), (1, 640)]),           # history clips at lower resolution + the current clip
    (128, [(1, 30), (2, 120), (3, 200)]),
    (24, [(4, 33), (1, 257)]),                      # seq % 128 != 0, tiles that cut through many frames
]


@pytest.mark.parametrize("text,clips", LAYOUTS)
def test_kv_schedule_is_the_transpose_and_matches_the_dense_mask(text, clips):
    g = torch.Generator().manual_seed(text + len(clips))
    seg, time = _pyramid_layout(g, 3, text, clips)
    batch, seq = seg.shape
    sched, _ = ops.attn_build_schedule(seg, time)
    kv = ops.attn_build_kv_schedule(sched, seq)
    tiles = (seq + 127) // 128
    assert kv.shape == sched.shape
    dense = _dense(seg, time)
    for b in range(batch):
        fwd = {}
        for qt in range(tiles):
            for e in sched[b, qt, 1:1 + int(sched[b, qt, 0])].tolist():
                fwd[(qt, e >> 1)] = e & 1
        back = {}
        for kt in range(tiles):
            n = int(kv[b, kt, 0])
            ent = kv[b, kt, 1:1 + n].tolist()
            assert [e >> 1 for e in ent] == sorted({e >> 1 for e in ent}), "q tiles strictly increasing"
            assert bool((kv[b, kt, 1 + n:] == 0).all())
            for e in ent:
                back[(e >> 1, kt)] = e & 1
        assert back == fwd
        # classes tile by tile against the dense definition: skipped = no allowed pair, unflagged = every pair of a full
        # 128 x 128 kv tile allowed, flagged = anything else with an allowed pair
        for qt in range(tiles):
            for kt in range(tiles):
                blk = dense[b, qt * 128:(qt + 1) * 128, kt * 128:(kt + 1) * 128]
                if not bool(blk.any()):
                    assert (qt, kt) not in back
                    continue
                assert (qt, kt) in back
                if back[(qt, kt)] == 0:
                    assert bool(blk.all()) and blk.shape[1] == 128


def _restated_stage_masks(sample, enc_mask, hidden_length, temporal_causal, patch=2):
    """F:320-350 restated: token ids (sample id + 1, 0 for padded text) equal, and with temporal causality the order ids
    (frame stamp of each clip's frames, consecutive over the stage's clips; text 0) non-increasing from q to kv."""
    num_stages = len(sample)
    real_bs, text_len = enc_mask.shape
    pad_bs = real_bs // num_stages
    text_ids = torch.arange(1, real_bs + 1)[:, None].repeat(1, text_len)
    text_ids[enc_mask == 0] = 0
    image_ids = torch.arange(1, real_bs + 1)[:, None].repeat(1, max(hidden_length))
    masks = []
    for i_p, length in enumerate(hidden_length):
        tok = torch.cat([text_ids[i_p::num_stages], image_ids[i_p::num_stages][:, :length]], dim=1)
        m = tok[:, :, None] == tok[:, None, :]
        if temporal_causal:
            order = [0] * text_len
            stamp = 0
            for clip in sample[i_p]:
                _, _, t, h, w = clip.shape
                for f in range(t):
                    order += [stamp + f] * ((h // patch) * (w // patch))
                stamp += t
            o = torch.tensor(order)[None].repeat(pad_bs, 1)
            m &= o[:, :, None] >= o[:, None, :]
        masks.append(m[:, None])
    return masks


class _StubDiT:
    """What stage_ids reads from the model: the pyramid order ids, restated (F:186-237, time coordinate only)."""

    def __init__(self, temporal_causal):
        self.use_temporal_causal = temporal_causal

    def _prepare_pyramid_image_ids(self, sample, batch_size, device):
        out = []
        for clips in sample:
            ids, stamp = [], 0
            for clip in clips:
                _, _, t, h, w = clip.shape
                for f in range(t):
                    ids += [stamp + f] * ((h // 2) * (w // 2))
                stamp += t
            tt = torch.tensor(ids, dtype=torch.float32)[None, :, None].repeat(batch_size, 1, 3)
            out.append(tt)
        return out


def _two_stage_sample(g, bs=2):
    # stage 0: low resolution, history clip + current; stage 1: higher resolution, two history clips + current
    s0 = [torch.randn(bs, 16, 2, 4, 8, generator=g), torch.randn(bs, 16, 1, 8, 16, generator=g)]
    s1 = [torch.randn(bs, 16, 1, 4, 8, generator=g), torch.randn(bs, 16, 2, 8, 16, generator=g),
          torch.randn(bs, 16, 1, 16, 32, generator=g)]
    enc_mask = torch.ones(2 * bs, 24, dtype=torch.long)
    enc_mask[0, 9:] = 0
    enc_mask[3, 17:] = 0
    return [s0, s1], enc_mask


@pytest.mark.parametrize("temporal_causal", [True, False])
def test_stage_ids_reproduce_the_dense_mask(temporal_causal):
    g = torch.Generator().manual_seed(5)
    sample, enc_mask = _two_stage_sample(g)
    hidden_length = [sum(c.shape[2] * (c.shape[3] // 2) * (c.shape[4] // 2) for c in clips) for clips in sample]
    ids = training.stage_ids(_StubDiT(temporal_causal), sample, enc_mask, hidden_length)
    want = _restated_stage_masks(sample, enc_mask, hidden_length, temporal_causal)
    assert len(ids) == 2
    for (seg, time), m in zip(ids, want):
        assert torch.equal(_dense(seg, time)[:, None], m)


def _reference_flux():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    return __import__("pyramid_dit.flux_modules", fromlist=["PyramidFluxTransformer"]).PyramidFluxTransformer


@pytest.mark.parametrize("temporal_causal", [True, False])
def test_wrapped_merge_input_of_the_reference_model(temporal_causal):
    """On the unmodified reference model: the wrapped merge_input returns one plan per stage whose seg / time give exactly
    the model's own dense masks (and the restatement of F:341-350), and everything else unchanged."""
    flux = _reference_flux()
    torch.manual_seed(0)
    model = flux(num_layers=1, num_single_layers=1, num_attention_heads=2, attention_head_dim=64, in_channels=64,
                 joint_attention_dim=32, pooled_projection_dim=16, use_temporal_causal=temporal_causal)
    g = torch.Generator().manual_seed(6)
    sample, enc_mask = _two_stage_sample(g)
    with torch.no_grad():
        ref_out = model.merge_input(sample, enc_mask.shape[1], enc_mask)
        training.install_training_attention(model)
        try:
            out = model.merge_input(sample, enc_mask.shape[1], enc_mask)
        finally:
            training.uninstall_training_attention(model)
        assert "merge_input" not in model.__dict__
    want = _restated_stage_masks(sample, enc_mask, ref_out[1], temporal_causal)
    for i_p, plan in enumerate(out[7]):
        assert isinstance(plan, training.StageAttentionPlan)
        got = _dense(plan.seg, plan.time)[:, None]
        assert torch.equal(got, ref_out[7][i_p]) and torch.equal(got, want[i_p])
    for i in (0, 8):
        for a, b in zip(out[i], ref_out[i]):
            assert torch.equal(a, b)
    assert list(out[1]) == list(ref_out[1])


def test_install_refuses_the_flash_path():
    flux = _reference_flux()
    model = flux(num_layers=1, num_single_layers=1, num_attention_heads=2, attention_head_dim=64, in_channels=64,
                 joint_attention_dim=32, pooled_projection_dim=16, use_flash_attn=True)
    with pytest.raises(ValueError, match="use_flash_attn"):
        training.install_training_attention(model)
    model = flux(num_layers=1, num_single_layers=1, num_attention_heads=2, attention_head_dim=32, in_channels=64,
                 joint_attention_dim=32, pooled_projection_dim=16, axes_dims_rope=[8, 12, 12])
    with pytest.raises(ValueError, match="head_dim"):
        training.install_training_attention(model)


def test_c_entries_reject_bad_descriptors():
    """Argument validation is host-side and happens before any CUDA call; pointers are dummies, never dereferenced."""
    from pyramid_flow_b200._lib import AttnBwdDesc, AttnDesc
    lib = _lib.load()
    dummy = 0x1000

    def err():
        return lib.pf_last_error().decode()

    a = AttnDesc()
    a.q = a.k = a.v = a.out = a.seg = a.time = a.tile_sched = a.lse = dummy
    a.batch, a.heads, a.seq, a.head_dim, a.ldo, a.sched_stride = 1, 2, 256, 64, 128, 3
    a.peer_count, a.peer_chunk_rows = 2, 128
    a.peer_out[0] = a.peer_out[1] = dummy
    assert lib.pf_attn_fwd_masked(C.byref(a), None) < 0 and "lse" in err()
    a.peer_count, a.q_row_begin = 0, 128
    assert lib.pf_attn_fwd_masked(C.byref(a), None) < 0 and "lse" in err()

    d = AttnBwdDesc()
    for f in ("q", "k", "v", "out", "dout", "lse", "seg", "time", "tile_sched", "kv_sched", "delta", "dq", "dk", "dv"):
        setattr(d, f, dummy)
    d.batch, d.heads, d.seq, d.head_dim, d.ldo, d.lddo, d.sched_stride, d.scale = 1, 2, 256, 32, 128, 128, 3, 0.125
    assert lib.pf_attn_bwd_masked(C.byref(d), None) < 0 and "head_dim" in err()
    d.head_dim, d.sched_stride = 64, 2
    assert lib.pf_attn_bwd_masked(C.byref(d), None) < 0 and "stride" in err()
    d.sched_stride, d.lddo = 3, 100
    assert lib.pf_attn_bwd_masked(C.byref(d), None) < 0 and "lddo" in err()
    d.lddo, d.kv_sched = 128, None
    assert lib.pf_attn_bwd_masked(C.byref(d), None) < 0 and "null" in err()
    assert lib.pf_attn_bwd_masked(None, None) < 0 and "null" in err()

    bad = torch.zeros(1, 3, 4, dtype=torch.int32)
    bad[0, 0, :2] = torch.tensor([1, 9 << 1])               # kv tile 9 of a 3-tile sequence
    out = torch.zeros_like(bad)
    assert lib.pf_attn_build_kv_schedule(bad.data_ptr(), 1, 300, 4, out.data_ptr()) < 0 and "range" in err()
    assert lib.pf_attn_build_kv_schedule(bad.data_ptr(), 1, 300, 3, out.data_ptr()) < 0 and "stride" in err()


def test_kv_schedule_refuses_a_kv_tile_named_twice():
    lib = _lib.load()
    bad = torch.zeros(1, 3, 4, dtype=torch.int32)
    bad[0, 0, :4] = torch.tensor([3, 1 << 1, 1 << 1, 1 << 1])    # q tile 0 names kv tile 1 three times
    out = torch.zeros_like(bad)
    assert lib.pf_attn_build_kv_schedule(bad.data_ptr(), 1, 300, 4, out.data_ptr()) < 0
    assert "more than once" in lib.pf_last_error().decode()


def test_c_entry_rejects_bad_batch_strides():
    from pyramid_flow_b200._lib import AttnBwdDesc
    lib = _lib.load()
    d = AttnBwdDesc()
    for f in ("q", "k", "v", "out", "dout", "lse", "seg", "time", "tile_sched", "kv_sched", "delta", "dq", "dk", "dv"):
        setattr(d, f, 0x1000)
    d.batch, d.heads, d.seq, d.head_dim, d.ldo, d.lddo, d.sched_stride, d.scale = 2, 2, 256, 64, 128, 128, 3, 0.125
    d.out_batch_stride, d.dout_batch_stride = 256 * 128, 0
    assert lib.pf_attn_bwd_masked(C.byref(d), None) < 0 and "batch stride" in lib.pf_last_error().decode()
    d.dout_batch_stride = 256 * 128 + 4
    assert lib.pf_attn_bwd_masked(C.byref(d), None) < 0 and "batch stride" in lib.pf_last_error().decode()


def test_attn_bwd_layout_rule():
    """Which dout views the backward takes as they are: a stage's slice of the single blocks' [attn | mlp] gradient (row
    stride D + mlp, batch stride total_len * (D + mlp)) is one of them; a row stride that is not a multiple of 8 is not."""
    wide = torch.zeros(2, 1072, 192 + 768, dtype=torch.bfloat16)
    view = wide[:, 232:, :192]
    assert view.stride() == (1072 * 960, 960, 1) and ops.attn_bwd_rows_ok(view)
    assert not ops.attn_bwd_rows_ok(torch.zeros(2, 10, 196, dtype=torch.bfloat16)[:, :, :192])
    assert not ops.attn_bwd_rows_ok(torch.zeros(2, 10, 192, dtype=torch.float32))
