"""The training-attention drop-in under an unmodified reference PyramidDiffusionMMDiT in a training step on the H100: three joint
blocks (the last one context_pre_only), temporal RoPE, temporal causality, gradient checkpointing, two stages with history
clips; fp32 and bf16 parameters."""
import copy

import pytest
import torch

from pyramid_flow_b200 import training
from tests.test_train_attn_gpu import DEV, _model_inputs, _train_step

pytestmark = pytest.mark.gpu


def _reference_mmdit():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    mmdit = __import__("pyramid_dit.mmdit_modules", fromlist=["PyramidDiffusionMMDiT"]).PyramidDiffusionMMDiT
    model = mmdit(num_layers=3, num_attention_heads=3, attention_head_dim=64, in_channels=16, caption_projection_dim=192,
                  joint_attention_dim=64, pooled_projection_dim=32, pos_embed_max_size=32, sample_size=64,
                  pos_embed_type="sincos", temp_pos_embed_type="rope", add_temp_pos_embed=True, use_flash_attn=False,
                  use_temporal_causal=True, use_gradient_checkpointing=True, gradient_checkpointing_ratio=0.5)
    assert model.transformer_blocks[-1].context_pre_only
    return model, ref_shim


def _errors(g, g32):
    num = torch.cat([(g[n] - g32[n]).flatten() for n in g32]).pow(2).sum().sqrt().item()
    return num / torch.cat([g32[n].flatten() for n in g32]).pow(2).sum().sqrt().item()


@pytest.mark.parametrize("params", ["fp32", "bf16"])
def test_reference_mmdit_training_step_with_installed_attention(params):
    model, ref_shim = _reference_mmdit()
    ref_shim.reinit_all_parameters(model, seed=7, std=0.05)
    model32 = copy.deepcopy(model).to(DEV).train()
    dtype = torch.float32 if params == "fp32" else torch.bfloat16
    model = model.to(DEV, dtype).train()
    inputs = _model_inputs()

    loss32, g32, _ = _train_step(model32, inputs, torch.float32, autocast=False)
    loss_sdpa, g_sdpa, peak_sdpa = _train_step(model, inputs, dtype, autocast=True)
    training.install_training_attention(model)
    try:
        loss_ours, g_ours, peak_ours = _train_step(model, inputs, dtype, autocast=True)
        loss_ours2, g_ours2, _ = _train_step(model, inputs, dtype, autocast=True)
    finally:
        training.uninstall_training_attention(model)
    loss_back, _, _ = _train_step(model, inputs, dtype, autocast=True)

    e_ours, e_sdpa = _errors(g_ours, g32), _errors(g_sdpa, g32)
    print(f"{params} parameters: loss fp32 {loss32.item():.6f}, bf16 SDPA {loss_sdpa.item():.6f}, installed {loss_ours.item():.6f}; "
          f"all gradients, relative error vs fp32: installed {e_ours:.3e}, SDPA {e_sdpa:.3e}; "
          f"peak memory SDPA {peak_sdpa / 2**20:.1f} MiB, installed {peak_ours / 2**20:.1f} MiB")
    assert set(g_ours) == set(g32) == set(g_sdpa) and len(g32) > 10
    assert e_ours <= 1.5 * e_sdpa
    for n in g32:
        d = g32[n].norm().item()
        if d > 0:
            eo, es = (g_ours[n] - g32[n]).norm().item() / d, (g_sdpa[n] - g32[n]).norm().item() / d
            assert eo <= 1.5 * max(es, 1e-3), (n, eo, es)
    assert abs(loss_ours - loss32) <= 1.5 * abs(loss_sdpa - loss32) + 1e-3 * abs(loss32)
    assert torch.equal(loss_ours, loss_ours2) and all(torch.equal(g_ours[n], g_ours2[n]) for n in g_ours)
    assert peak_ours <= peak_sdpa
    assert torch.equal(loss_back, loss_sdpa), "after uninstall the model runs the SDPA path again"
