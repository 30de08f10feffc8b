"""Trainable masked attention on the H100: forward log-sum-exp, gradients against fp32 autograd, determinism, and the drop-in
under the unmodified reference PyramidFluxTransformer in a training step."""
import copy

import pytest
import torch
import torch.nn.functional as F

from pyramid_flow_b200 import ops, training

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _layout(g, batch, text, clips, causal=True):
    segs, times = [], []
    for b in range(batch):
        valid = text - 7 * (b + 1) if text > 16 else text
        seg = [1] * valid + [0] * (text - valid)
        time = [0] * text
        stamp = 0
        for t, n in clips:
            for f in range(t):
                seg += [1] * n
                time += [(stamp + f) if causal else 0] * n
            stamp += t
        segs.append(seg)
        times.append(time)
    return torch.tensor(segs, dtype=torch.int32), torch.tensor(times, dtype=torch.int32)


def _dense(seg, time):
    return (seg[:, :, None] == seg[:, None, :]) & (time[:, :, None] >= time[:, None, :])


CASES = {
    # B = 2, 3 heads; text padded differently per sample; history clips + the current clip; seq % 128 != 0
    "pyramid": (128, [(2, 48), (1, 96), (1, 384)], True),
    # 40-token frames: every q tile meets only partial kv tiles
    "all_partial": (24, [(6, 40)], True),
    # no temporal causality: the mask is the text padding only
    "no_causal": (77, [(1, 60), (2, 150)], False),
}


def _inputs(case, seed=0):
    text, clips, causal = CASES[case]
    g = torch.Generator().manual_seed(seed)
    seg, time = _layout(g, 2, text, clips, causal)
    b, s = seg.shape
    q, k, v = (torch.randn(b, 3, s, 64, generator=g).to(DEV, torch.bfloat16) for _ in range(3))
    dout = torch.randn(b, 3, s, 64, generator=g).to(DEV, torch.bfloat16)
    return seg, time, q, k, v, dout


def _rel_rms(x, ref):
    return ((x.float() - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()


def test_forward_lse_keeps_the_output_bits():
    seg, time, q, k, v, _ = _inputs("pyramid")
    b, h, s, _ = q.shape
    sched, _ = ops.attn_build_schedule(seg, time)
    segd, timed, schedd = seg.to(DEV), time.to(DEV), sched.to(DEV)
    out0 = torch.zeros(b, s, h * 64, dtype=torch.bfloat16, device=DEV)
    out1 = torch.zeros_like(out0)
    lse = torch.zeros(b, h, s, dtype=torch.float32, device=DEV)
    ops.attn_fwd(q, k, v, out0, segd, timed, schedd, 0.125)
    ops.attn_fwd(q, k, v, out1, segd, timed, schedd, 0.125, lse=lse)
    torch.cuda.synchronize()
    assert torch.equal(out0, out1)
    scores = (q.float() @ k.float().transpose(-1, -2)) * 0.125
    scores = scores.masked_fill(~_dense(seg, time)[:, None].to(DEV), float("-inf"))
    want = torch.logsumexp(scores, dim=-1)
    rel = ((lse - want).abs() / want.abs().clamp_min(1e-6)).max().item()
    print(f"lse vs fp32 logsumexp: max relative error {rel:.2e}")
    assert rel <= 1e-4


@pytest.mark.parametrize("case", list(CASES))
def test_gradients_against_fp32_autograd(case):
    seg, time, q, k, v, dout = _inputs(case)
    b, h, s, _ = q.shape
    mask = _dense(seg, time)[:, None].to(DEV)

    # fp32 autograd of softmax attention with the dense mask
    q32, k32, v32 = (t.float().requires_grad_() for t in (q, k, v))
    p = torch.softmax((q32 @ k32.transpose(-1, -2) * 0.125).masked_fill(~mask, float("-inf")), dim=-1)
    o32 = p @ v32
    o32.backward(dout.float())
    ref = dict(out=o32.detach(), dq=q32.grad, dk=k32.grad, dv=v32.grad)

    # bf16 SDPA with the same dense mask (what the reference runs)
    qs, ks, vs = (t.clone().requires_grad_() for t in (q, k, v))
    os_ = F.scaled_dot_product_attention(qs, ks, vs, attn_mask=mask)
    os_.backward(dout)
    sdpa = dict(out=os_.detach(), dq=qs.grad, dk=ks.grad, dv=vs.grad)

    def ours():
        qo, ko, vo = (t.clone().requires_grad_() for t in (q, k, v))
        out = training.masked_attention(qo, ko, vo, seg.to(DEV), time.to(DEV))
        out.backward(dout.transpose(1, 2).reshape(b, s, h * 64))
        return dict(out=out.detach().view(b, s, h, 64).transpose(1, 2), dq=qo.grad, dk=ko.grad, dv=vo.grad)

    first, second = ours(), ours()
    torch.cuda.synchronize()
    for name in ("out", "dq", "dk", "dv"):
        e_ours, e_sdpa = _rel_rms(first[name], ref[name]), _rel_rms(sdpa[name], ref[name])
        print(f"{case} {name}: relative RMS error vs fp32 {e_ours:.3e} (bf16 SDPA {e_sdpa:.3e}, ratio {e_ours / e_sdpa:.2f})")
        assert torch.isfinite(first[name]).all()
        assert e_ours <= 1.5 * e_sdpa, (case, name, e_ours, e_sdpa)
        assert torch.equal(first[name], second[name]), f"{case} {name}: two runs differ"


def _reference_flux():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    return __import__("pyramid_dit.flux_modules", fromlist=["PyramidFluxTransformer"]).PyramidFluxTransformer, ref_shim


def _model_inputs(bs=2):
    g = torch.Generator().manual_seed(11)
    # two stages of the temporal pyramid: history clips at lower resolution + the current clip
    sample = [[torch.randn(bs, 16, 2, 8, 16, generator=g), torch.randn(bs, 16, 1, 16, 32, generator=g)],
              [torch.randn(bs, 16, 1, 8, 16, generator=g), torch.randn(bs, 16, 2, 16, 32, generator=g),
               torch.randn(bs, 16, 1, 32, 64, generator=g)]]
    enc = torch.randn(2 * bs, 40, 64, generator=g)
    mask = torch.ones(2 * bs, 40, dtype=torch.long)
    mask[0, 13:] = 0
    mask[3, 29:] = 0
    pooled = torch.randn(2 * bs, 32, generator=g)
    t = torch.tensor([900.0, 300.0] * bs)
    targets = [torch.randn(bs, 16, 1, 16, 32, generator=g), torch.randn(bs, 16, 1, 32, 64, generator=g)]
    return sample, enc, mask, pooled, t, targets


def _train_step(model, inputs, dtype, autocast):
    sample, enc, mask, pooled, t, targets = inputs
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()      # what earlier steps left alive (their gradient copies) is not this step's
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        preds = model(sample=[[c.to(DEV, dtype) for c in clips] for clips in sample], encoder_hidden_states=enc.to(DEV, dtype),
                      encoder_attention_mask=mask.to(DEV), pooled_projections=pooled.to(DEV, dtype), timestep_ratio=t.to(DEV, dtype))
        loss = sum(((p.float() - y.to(DEV)) ** 2).mean() for p, y in zip(preds, targets))
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    grads = {n: p.grad.detach().float().clone() for n, p in model.named_parameters() if p.grad is not None}
    return loss.detach().float(), grads, peak


def test_reference_training_step_with_installed_attention():
    flux, ref_shim = _reference_flux()
    cfg = dict(num_layers=2, num_single_layers=2, num_attention_heads=3, attention_head_dim=64, in_channels=64,
               joint_attention_dim=64, pooled_projection_dim=32, use_temporal_causal=True, use_gradient_checkpointing=True,
               gradient_checkpointing_ratio=1.0)
    model = flux(**cfg)
    ref_shim.reinit_all_parameters(model, seed=3, std=0.05)
    model = model.to(DEV).train()
    model32 = copy.deepcopy(model)
    inputs = _model_inputs()

    loss32, g32, _ = _train_step(model32, inputs, torch.float32, autocast=False)
    loss_sdpa, g_sdpa, peak_sdpa = _train_step(model, inputs, torch.float32, autocast=True)
    training.install_training_attention(model)
    loss_ours, g_ours, peak_ours = _train_step(model, inputs, torch.float32, autocast=True)
    loss_ours2, g_ours2, _ = _train_step(model, inputs, torch.float32, autocast=True)
    training.uninstall_training_attention(model)
    loss_back, _, _ = _train_step(model, inputs, torch.float32, autocast=True)

    print(f"loss fp32 {loss32.item():.6f}, bf16 SDPA {loss_sdpa.item():.6f}, bf16 installed {loss_ours.item():.6f}")
    print(f"peak memory: SDPA path {peak_sdpa / 2**20:.1f} MiB, installed {peak_ours / 2**20:.1f} MiB")
    assert set(g_ours) == set(g32) == set(g_sdpa) and len(g32) > 10
    num = lambda gs: torch.cat([(gs[n] - g32[n]).flatten() for n in g32]).pow(2).sum().sqrt().item()
    den = torch.cat([g32[n].flatten() for n in g32]).pow(2).sum().sqrt().item()
    e_ours, e_sdpa = num(g_ours) / den, num(g_sdpa) / den
    print(f"all parameter gradients, relative error vs fp32: installed {e_ours:.3e}, SDPA {e_sdpa:.3e}")
    assert e_ours <= 1.5 * e_sdpa
    worst = 0.0
    for n in g32:
        d = g32[n].norm().item()
        if d == 0:
            continue
        eo, es = (g_ours[n] - g32[n]).norm().item() / d, (g_sdpa[n] - g32[n]).norm().item() / d
        worst = max(worst, eo / max(es, 1e-3))
        assert eo <= 1.5 * max(es, 1e-3), (n, eo, es)
    print(f"worst per-parameter ratio (installed / max(SDPA, 1e-3)): {worst:.2f}")
    assert abs(loss_ours - loss32) <= 1.5 * abs(loss_sdpa - loss32) + 1e-6 * abs(loss32)
    assert torch.equal(loss_ours, loss_ours2) and all(torch.equal(g_ours[n], g_ours2[n]) for n in g_ours)
    assert peak_ours <= peak_sdpa
    assert torch.equal(loss_back, loss_sdpa), "after uninstall the model runs the SDPA path again"


def test_install_refuses_the_flash_path_model():
    flux, _ = _reference_flux()
    model = flux(num_layers=1, num_single_layers=1, num_attention_heads=2, attention_head_dim=64, in_channels=64,
                 joint_attention_dim=32, pooled_projection_dim=16, use_flash_attn=True).to(DEV)
    with pytest.raises(ValueError):
        training.install_training_attention(model)


def test_gradients_through_the_single_block_concatenation(monkeypatch):
    """The single blocks concatenate the stages' attention outputs along the sequence and then with the MLP branch along the
    features (B:596-604, B:936): each stage's output gradient arrives as a view whose batch stride is not seq * row stride.
    Gradients must still match fp32 autograd as closely as bf16 SDPA's do."""
    g = torch.Generator().manual_seed(4)
    b, h, mlp = 2, 3, 256
    stages = [_layout(g, b, 24, [(2, 40), (1, 96)]), _layout(g, b, 40, [(1, 40), (2, 96), (1, 200)])]
    qkv = [tuple(torch.randn(b, h, seg.shape[1], 64, generator=g).to(DEV, torch.bfloat16) for _ in range(3)) for seg, _ in stages]
    total = sum(seg.shape[1] for seg, _ in stages)
    mlp_branch = torch.randn(b, total, mlp, generator=g).to(DEV, torch.bfloat16)
    weight = torch.randn(b, total, h * 64 + mlp, generator=g).to(DEV)

    def run(attn, dtype):
        leaves, outs = [], []
        for (seg, time), (q, k, v) in zip(stages, qkv):
            q, k, v = (t.to(dtype).clone().requires_grad_() for t in (q, k, v))
            leaves.append((q, k, v))
            outs.append(attn(q, k, v, seg, time))
        joint = torch.cat([torch.cat(outs, dim=1), mlp_branch.to(outs[0].dtype)], dim=2)        # B:936
        (joint.float() * weight).sum().backward()
        return [t.grad.float() for trio in leaves for t in trio]

    def dense_attn(q, k, v, seg, time):
        mask = _dense(seg, time)[:, None].to(DEV)
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        return o.transpose(1, 2).flatten(2, 3)

    seen = []
    real_bwd = ops.attn_bwd

    def recording_bwd(q, k, v, out, dout, *args, **kw):
        seen.append((tuple(dout.shape), dout.stride()))
        return real_bwd(q, k, v, out, dout, *args, **kw)

    monkeypatch.setattr(ops, "attn_bwd", recording_bwd)
    ours = run(lambda q, k, v, seg, time: training.masked_attention(q, k, v, seg.to(DEV), time.to(DEV)), torch.bfloat16)
    monkeypatch.undo()
    ref = run(dense_attn, torch.float32)
    sdpa = run(dense_attn, torch.bfloat16)
    torch.cuda.synchronize()
    print(f"dout layouts reaching the backward (shape, strides): {seen}")
    assert len(seen) == 2 and all(st[0] != shp[1] * st[1] for shp, st in seen), "expected strided stage views of the gradient"
    for i, (o, r, s_) in enumerate(zip(ours, ref, sdpa)):
        e_ours, e_sdpa = _rel_rms(o, r), _rel_rms(s_, r)
        print(f"stage {i // 3} {'qkv'[i % 3]}: relative RMS error vs fp32 {e_ours:.3e} (bf16 SDPA {e_sdpa:.3e})")
        assert e_ours <= 1.5 * e_sdpa, (i, e_ours, e_sdpa)


def test_reference_training_step_with_bf16_parameters():
    """The model in bf16 (as FSDP's bf16 mixed precision or a bf16 load gives it): q / k / v reach the attention in bf16 and
    the single blocks' output gradients reach the backward as strided views."""
    flux, ref_shim = _reference_flux()
    cfg = dict(num_layers=2, num_single_layers=2, num_attention_heads=3, attention_head_dim=64, in_channels=64,
               joint_attention_dim=64, pooled_projection_dim=32, use_temporal_causal=True, use_gradient_checkpointing=True,
               gradient_checkpointing_ratio=1.0)
    model = flux(**cfg)
    ref_shim.reinit_all_parameters(model, seed=5, std=0.05)
    model32 = copy.deepcopy(model).to(DEV).train()
    model = model.to(DEV, torch.bfloat16).train()
    inputs = _model_inputs()
    loss32, g32, _ = _train_step(model32, inputs, torch.float32, autocast=False)
    loss_sdpa, g_sdpa, _ = _train_step(model, inputs, torch.bfloat16, autocast=True)
    training.install_training_attention(model)
    try:
        loss_ours, g_ours, _ = _train_step(model, inputs, torch.bfloat16, autocast=True)
    finally:
        training.uninstall_training_attention(model)
    num = lambda gs: torch.cat([(gs[n] - g32[n]).flatten() for n in g32]).pow(2).sum().sqrt().item()
    den = torch.cat([g32[n].flatten() for n in g32]).pow(2).sum().sqrt().item()
    e_ours, e_sdpa = num(g_ours) / den, num(g_sdpa) / den
    print(f"bf16 parameters: loss fp32 {loss32.item():.6f}, SDPA {loss_sdpa.item():.6f}, installed {loss_ours.item():.6f}; "
          f"all gradients, relative error vs fp32: installed {e_ours:.3e}, SDPA {e_sdpa:.3e}")
    assert e_ours <= 1.5 * e_sdpa
    assert abs(loss_ours - loss32) <= 1.5 * abs(loss_sdpa - loss32) + 1e-3 * abs(loss32)
