"""Host side of the varlen (flash path) training attention, no GPU: the plan the wrapped merge_input builds from the unmodified
reference miniFLUX's indices / seqlens_in_batch, install / uninstall on the flash processors, the refusals, and the argument
checks of the C entries."""
import ctypes as C

import pytest
import torch

from pyramid_flow_b200 import _lib, training


def _reference_flux():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    return __import__("pyramid_dit.flux_modules", fromlist=["PyramidFluxTransformer"]).PyramidFluxTransformer


def _small(flux, **kw):
    cfg = dict(num_layers=1, num_single_layers=1, num_attention_heads=2, attention_head_dim=64, in_channels=64,
               joint_attention_dim=32, pooled_projection_dim=16, use_flash_attn=True)
    cfg.update(kw)
    return flux(**cfg)


def _sample(g, n_stages, bs=2, text=24):
    """A t2i / full-sequence t2v pyramid: one clip per stage at rising resolution; prompts padded differently per row
    (one row with all tokens valid, one with a single valid token)."""
    sizes = [(1, 4, 8), (2, 8, 16), (1, 16, 32)][:n_stages]
    sample = [[torch.randn(bs, 16, t, h, w, generator=g)] for t, h, w in sizes]
    mask = torch.ones(n_stages * bs, text, dtype=torch.long)
    for r in range(n_stages * bs):
        mask[r, [text, 1, 9, 17, 5, 13][r % 6]:] = 0
    return sample, mask


@pytest.mark.parametrize("n_stages", [2, 3])
def test_wrapped_merge_input_builds_the_reference_layout(n_stages):
    flux = _reference_flux()
    torch.manual_seed(0)
    model = _small(flux)
    sample, mask = _sample(torch.Generator().manual_seed(n_stages), n_stages)
    text = mask.shape[1]
    with torch.no_grad():
        ref = model.merge_input(sample, text, mask)
        training.install_varlen_training_attention(model)
        try:
            out = model.merge_input(sample, text, mask)
        finally:
            training.uninstall_training_attention(model)
    assert "merge_input" not in model.__dict__
    plan = out[6]
    assert isinstance(plan, training.VarlenAttentionPlan) and ref[7] is None and out[7] is None
    stage_len = [text + n for n in ref[1]]
    assert plan.stage_len == stage_len and plan.batch == 2
    # the row map enumerates each stage's indices, in the order of the reference's torch.cat(qkv_list)
    pad0, want = 0, []
    for st, length in zip(ref[6], stage_len):
        want.append(st["indices"] + pad0)
        pad0 += 2 * length
    want = torch.cat(want)
    assert torch.equal(plan.row_map.long(), want)
    assert torch.equal(plan.pad_map[plan.row_map.long()].long(), torch.arange(want.numel()))
    assert int((plan.pad_map >= 0).sum()) == want.numel() and plan.pad_map.numel() == pad0
    # seg numbers the (stage, batch) sequences: its run lengths are the cu_seqlens of the reference's flash call
    seqlens = torch.cat([st["seqlens_in_batch"] for st in ref[6]])
    cu = torch.nn.functional.pad(torch.cumsum(seqlens, dim=0, dtype=torch.int32), (1, 0))
    assert torch.equal(plan.cu_seqlens, cu) and plan.max_seqlen == int(seqlens.max())
    _, runs = torch.unique_consecutive(plan.seg[0], return_counts=True)
    assert torch.equal(runs.to(torch.int32), seqlens) and torch.equal(plan.seg[0].unique(), torch.arange(1, seqlens.numel() + 1,
                                                                                                          dtype=torch.int32))
    assert not bool(plan.time.any())
    for i in (0, 2, 3, 4, 5):
        assert out[i] == ref[i] if i != 0 else all(torch.equal(a, b) for a, b in zip(out[0], ref[0]))
    assert list(out[1]) == list(ref[1])
    assert all(torch.equal(a, b) for a, b in zip(out[8], ref[8]))
    # a second call with the same layout reuses the plan
    with torch.no_grad():
        training.install_varlen_training_attention(model)
        try:
            assert model.merge_input(sample, text, mask)[6] is plan
        finally:
            training.uninstall_training_attention(model)


def test_install_replaces_every_flash_callable_and_uninstall_restores_them():
    flux = _reference_flux()
    model = _small(flux, num_layers=2, num_single_layers=3)
    procs = [m.processor for m in model.modules() if type(getattr(m, "processor", None)).__name__ in
             ("FluxAttnProcessor2_0", "FluxSingleAttnProcessor2_0")]
    assert len(procs) == 5
    before = [p.varlen_flash_attn for p in procs]
    training.install_varlen_training_attention(model)
    installed = [p.varlen_flash_attn for p in procs]
    training.install_varlen_training_attention(model)          # idempotent
    assert [p.varlen_flash_attn for p in procs] == installed
    assert all(type(f).__module__ == training.__name__ for f in installed)
    assert [type(f).__name__ for f in installed] == ["_VarlenJointAttention"] * 2 + ["_VarlenSingleAttention"] * 3
    assert "merge_input" in model.__dict__
    with pytest.raises(TypeError, match="VarlenAttentionPlan"):
        installed[0](*([torch.zeros(1, 1, 1, 64)] * 6), 1, 0.125, [1], None, [{"indices": None}])
    with pytest.raises(TypeError, match="VarlenAttentionPlan"):
        installed[2](*([torch.zeros(1, 1, 1, 64)] * 3), 1, 0.125, [1], None, None)
    training.uninstall_training_attention(model)
    assert [p.varlen_flash_attn for p in procs] == before and "merge_input" not in model.__dict__
    assert getattr(model, "_pf_training_attention", None) is None


def test_install_refusals():
    flux = _reference_flux()
    with pytest.raises(ValueError, match="install_training_attention"):
        training.install_varlen_training_attention(_small(flux, use_flash_attn=False))
    with pytest.raises(ValueError, match="head_dim"):
        training.install_varlen_training_attention(_small(flux, attention_head_dim=32, axes_dims_rope=[8, 12, 12]))
    # the existing drop-in still refuses the flash model, naming the flash path
    with pytest.raises(ValueError, match="use_flash_attn"):
        training.install_training_attention(_small(flux))


def test_install_refuses_sequence_parallelism(monkeypatch):
    flux = _reference_flux()
    model = _small(flux)
    import sys
    mod = sys.modules[type(model).__module__]
    monkeypatch.setattr(mod, "is_sequence_parallel_initialized", lambda: True)
    with pytest.raises(ValueError, match="sequence parallel"):
        training.install_varlen_training_attention(model)


def test_install_refuses_the_mmdit():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    mmdit = __import__("pyramid_dit.mmdit_modules", fromlist=["PyramidDiffusionMMDiT"]).PyramidDiffusionMMDiT
    model = mmdit(sample_size=16, patch_size=2, in_channels=16, num_layers=1, attention_head_dim=64, num_attention_heads=2,
                  caption_projection_dim=128, joint_attention_dim=64, pooled_projection_dim=32, pos_embed_max_size=32,
                  use_flash_attn=False, use_temporal_causal=True)
    with pytest.raises(ValueError, match="MMDiT"):
        training.install_varlen_training_attention(model)


def test_plan_rejects_inconsistent_indices():
    ok = ([torch.tensor([0, 1, 5, 6, 7])], [torch.tensor([2, 3], dtype=torch.int32)])
    assert training.varlen_plan(*ok, 2, [4]).total == 5
    with pytest.raises(ValueError, match="seqlens_in_batch"):
        training.varlen_plan([torch.tensor([0, 1, 5, 6, 7])], [torch.tensor([3, 2], dtype=torch.int32)], 2, [4])
    with pytest.raises(ValueError, match="seqlens_in_batch"):
        training.varlen_plan([torch.tensor([0, 1, 5, 6, 8])], [torch.tensor([2, 3], dtype=torch.int32)], 2, [4])
    with pytest.raises(ValueError, match="at least one row"):
        training.varlen_plan([torch.tensor([4, 5])], [torch.tensor([0, 2], dtype=torch.int32)], 2, [4])


def test_c_entries_reject_bad_descriptors_without_a_launch():
    """Argument validation is host-side and happens before any CUDA call; pointers are dummies, never dereferenced."""
    from pyramid_flow_b200._lib import AttnVarlenPackDesc, AttnVarlenUnpackDesc
    lib = _lib.load()
    dummy = 0x1000

    def layout(lay):
        lay.batch, lay.heads, lay.head_dim, lay.text_len, lay.src_rows, lay.n_stages, lay.total = 2, 3, 64, 24, 300, 2, 400
        lay.stage_len[0], lay.stage_len[1], lay.stage_row0[0], lay.stage_row0[1] = 124, 224, 0, 100
        lay.row_map = lay.pad_map = dummy

    def pack():
        d = AttnVarlenPackDesc()
        layout(d.layout)
        for i in range(3):
            d.video[i] = d.text[i] = d.packed[i] = dummy
            for j, st in enumerate((300 * 192, 192, 64)):
                d.video_strides[i][j] = st
            for j, st in enumerate((24 * 192, 192, 64)):
                d.text_strides[i][j] = st
        return d

    def unpack():
        d = AttnVarlenUnpackDesc()
        layout(d.layout)
        d.video = d.text = d.packed = dummy
        d.video_strides[0], d.video_strides[1], d.text_strides[0], d.text_strides[1], d.ld_packed = 300 * 192, 192, 24 * 192, 192, 192
        return d

    launches = lib.pf_launch_count()
    bad = []
    d = pack(); d.layout.head_dim = 128; bad.append((d, "head_dim"))
    d = pack(); d.layout.stage_row0[1] = 200; bad.append((d, "outside"))
    d = pack(); d.layout.stage_len[0] = 24; bad.append((d, "outside"))
    d = pack(); d.layout.n_stages = 9; bad.append((d, "n_stages"))
    d = pack(); d.layout.total = 700; bad.append((d, "exceeds"))
    d = pack(); d.layout.pad_map = None; bad.append((d, "pad_map"))
    d = pack(); d.video_strides[1][1] = 196; bad.append((d, "multiple of 8"))
    d = pack(); d.text[2] = dummy + 8; bad.append((d, "aligned"))
    d = pack(); d.freqs[1], d.freqs_batch_stride[1], d.freqs_row_stride[1] = dummy, 224 * 128, 64; bad.append((d, "freqs[1]"))
    for d, what in bad:
        for entry in (lib.pf_attn_varlen_pack, lib.pf_attn_varlen_pack_bwd):
            assert entry(C.byref(d), None) < 0 and what in lib.pf_last_error().decode(), (what, lib.pf_last_error())
    bad = []
    d = unpack(); d.ld_packed = 100; bad.append((d, "ld_packed"))
    d = unpack(); d.video_strides[1] = 100; bad.append((d, "video strides"))
    d = unpack(); d.text_f32 = 3; bad.append((d, "text_f32"))
    d = unpack(); d.layout.row_map = dummy + 2; bad.append((d, "row_map"))
    for d, what in bad:
        for entry in (lib.pf_attn_varlen_unpack, lib.pf_attn_varlen_unpack_bwd):
            assert entry(C.byref(d), None) < 0 and what in lib.pf_last_error().decode(), (what, lib.pf_last_error())
    for entry in (lib.pf_attn_varlen_pack, lib.pf_attn_varlen_unpack):
        assert entry(None, None) < 0 and "null" in lib.pf_last_error().decode()
    assert lib.pf_launch_count() == launches
