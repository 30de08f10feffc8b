"""The training-attention drop-in on an unmodified reference PyramidDiffusionMMDiT, host side (no GPU): the wrapped merge_input's
plans against the model's own dense masks, which attention callables the install replaces, and what it refuses."""
import sys

import pytest
import torch

from pyramid_flow_b200 import training
from tests.test_train_attn_cpu import _dense, _restated_stage_masks, _two_stage_sample


def _reference_mmdit():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    return __import__("pyramid_dit.mmdit_modules", fromlist=["PyramidDiffusionMMDiT"]).PyramidDiffusionMMDiT


def _small(mmdit, **kw):
    cfg = dict(num_layers=3, num_attention_heads=2, attention_head_dim=64, in_channels=16, caption_projection_dim=128,
               joint_attention_dim=32, pooled_projection_dim=16, pos_embed_max_size=24, sample_size=32, pos_embed_type="sincos",
               temp_pos_embed_type="rope", add_temp_pos_embed=True, use_flash_attn=False, use_temporal_causal=True)
    cfg.update(kw)
    return mmdit(**cfg)


@pytest.mark.parametrize("temporal_causal", [True, False])
def test_wrapped_merge_input_of_the_reference_mmdit(temporal_causal):
    """Two stages with history clips and padded prompts: one plan per stage whose seg / time give exactly the model's own
    dense masks (M:369-378) and their restatement; everything else merge_input returns is unchanged."""
    mmdit = _reference_mmdit()
    torch.manual_seed(0)
    model = _small(mmdit, use_temporal_causal=temporal_causal)
    sample, enc_mask = _two_stage_sample(torch.Generator().manual_seed(6))
    with torch.no_grad():
        ref_out = model.merge_input(sample, enc_mask.shape[1], enc_mask)
        training.install_training_attention(model)
        try:
            out = model.merge_input(sample, enc_mask.shape[1], enc_mask)
        finally:
            training.uninstall_training_attention(model)
        assert "merge_input" not in model.__dict__
    want = _restated_stage_masks(sample, enc_mask, ref_out[1], temporal_causal)
    assert len(out[7]) == len(sample) == 2
    for i_p, plan in enumerate(out[7]):
        assert isinstance(plan, training.StageAttentionPlan)
        got = _dense(plan.seg, plan.time)[:, None]
        assert torch.equal(got, ref_out[7][i_p]) and torch.equal(got, want[i_p])
    for i in (0, 8):
        for a, b in zip(out[i], ref_out[i]):
            assert torch.equal(a, b)
    assert list(out[1]) == list(ref_out[1])


def test_install_replaces_every_joint_attention_and_uninstall_restores_them():
    mmdit = _reference_mmdit()
    model = _small(mmdit)
    blocks = model.transformer_blocks
    assert blocks[-1].context_pre_only and not blocks[0].context_pre_only
    before = [b.attn.var_len_attn for b in blocks]
    training.install_training_attention(model)
    training.install_training_attention(model)                     # idempotent
    assert all(isinstance(b.attn.var_len_attn, training._JointAttention) for b in blocks)
    training.uninstall_training_attention(model)
    assert [b.attn.var_len_attn for b in blocks] == before
    assert "merge_input" not in model.__dict__ and not hasattr(model, "_pf_training_attention")


def test_install_refuses_what_it_does_not_replace(monkeypatch):
    mmdit = _reference_mmdit()
    with pytest.raises(ValueError, match="use_flash_attn"):
        training.install_training_attention(_small(mmdit, use_flash_attn=True, use_temporal_causal=False))
    with pytest.raises(ValueError, match="head_dim"):
        training.install_training_attention(_small(mmdit, attention_head_dim=32, caption_projection_dim=64))
    model = _small(mmdit)
    monkeypatch.setattr(sys.modules[type(model).__module__], "is_sequence_parallel_initialized", lambda: True)
    with pytest.raises(ValueError, match="sequence parallel"):
        training.install_training_attention(model)
    assert not hasattr(model, "_pf_training_attention")
