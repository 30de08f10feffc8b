"""Parity at BASELINE.json's FULL sizes (768p, unit 30 / stage 2: B=2, S=15488, D=1920, 30 heads) on an H100.
The fp32 oracle is too slow for 24 blocks at this size on the CPU, so it runs on the same GPU in fp32 (TF32 off), with the
attention evaluated a few heads at a time to bound memory; plus size-independent properties of the attention kernel."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _full_inputs(gen):
    shapes = [(2, 16, 28, 24, 40), (2, 16, 1, 48, 80), (2, 16, 1, 96, 160), (2, 16, 1, 96, 160)]
    clips = [torch.randn(s, generator=gen).bfloat16().float() for s in shapes]
    enc = (torch.randn(2, 128, 4096, generator=gen) * 0.2).bfloat16().float()
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[0, 77:] = 0
    pooled = torch.randn(2, 768, generator=gen)
    return clips, enc, mask, pooled, torch.tensor([3.0, 3.0])


def test_full_size_step_two_plus_two_blocks_matches_oracle():
    from oracle import flux_oracle as FO
    from pyramid_flow_b200.dit import B200FluxTransformer, FluxConfigB200
    kw = dict(num_layers=2, num_single_layers=2)
    cfg = FO.FluxConfig(**kw)
    params = FO.synthetic_flux_params(cfg, seed=5)
    clips, enc, mask, pooled, t = _full_inputs(torch.Generator().manual_seed(9))
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from torch.nn.attention import SDPBackend, sdpa_kernel
    FO.HEAD_CHUNK = 3
    try:
        with torch.no_grad(), sdpa_kernel(SDPBackend.MATH):
            pd = {k: v.to(dev) for k, v in params.items()}
            ref = FO.flux_forward(pd, cfg, [c.to(dev) for c in clips], t.to(dev), enc.to(dev), mask, pooled.to(dev)).float().cpu()
            del pd
    finally:
        FO.HEAD_CHUNK = 0
    torch.cuda.empty_cache()
    model = B200FluxTransformer(FluxConfigB200(**kw), params, device=dev)
    out = model(sample=[[c.to(dev) for c in clips]], timestep_ratio=t.to(dev), encoder_hidden_states=enc.to(dev),
                encoder_attention_mask=mask.to(dev), pooled_projections=pooled.to(dev))[0].float().cpu()
    assert model.last_plan.seq == 15488
    err, mse = (out - ref).abs().max().item(), ((out - ref) ** 2).mean().item()
    print(f"full-size (S=15488, 2+2 blocks): max_abs {err:.3e} mse {mse:.3e} |v| mean {ref.abs().mean():.3f}")
    assert err < 1.3e-2 and mse < 5.7e-6


def test_attention_full_size_sampled_rows_and_properties():
    """S=15488, 30 heads: (1) sampled query rows vs an fp32 softmax over the full kv range with the dense mask definition;
    (2) linearity in V; (3) rows are convex combinations (constant V -> constant out)."""
    from pyramid_flow_b200 import ops
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    B, H = 2, 30
    lens = [128 + 240] + [240] * 27 + [960, 3840, 3840]
    tim = torch.cat([torch.full((n,), float(i)) for i, n in enumerate(lens)]).int()[None].repeat(B, 1)
    S = tim.shape[1]
    seg = torch.ones(B, S, dtype=torch.int32)
    seg[0, 90:128] = 0
    q = torch.randn(B, H, S, 64, device=dev).bfloat16()
    k = torch.randn(B, H, S, 64, device=dev).bfloat16()
    v1 = torch.randn(B, H, S, 64, device=dev).bfloat16()
    v2 = torch.randn(B, H, S, 64, device=dev).bfloat16()
    sched, pairs = ops.attn_build_schedule(seg, tim)
    ps = ops.attn_build_pair_schedule(sched, S, seg, tim).to(dev)
    sd, td, scd = seg.to(dev), tim.to(dev), sched.to(dev)

    def run(v):
        out = torch.zeros(B, S, H * 64, device=dev, dtype=torch.bfloat16)
        ops.attn_fwd(q, k, v, out, sd, td, scd, 0.125, pair_sched=ps)
        return out.float().view(B, S, H, 64)

    o1, o2, o12 = run(v1), run(v2), run((v1.float() + v2.float()).bfloat16())
    # (1) sampled rows, every frame boundary represented
    rows = torch.tensor([0, 50, 100, 127, 128, 367, 368, 5000, 6847, 6848, 7807, 7808, 11647, 11648, 15487], device=dev)
    for b in range(B):
        allowed = (sd[b][rows][:, None] == sd[b][None, :]) & (td[b][rows][:, None] >= td[b][None, :])      # [R, S]
        sc = torch.einsum("hrd,hsd->hrs", q[b][:, rows].float(), k[b].float()) * 0.125
        sc = sc.masked_fill(~allowed[None], float("-inf"))
        ref = torch.einsum("hrs,hsd->rhd", torch.softmax(sc, dim=-1), v1[b].float())
        assert (o1[b][rows] - ref).abs().max().item() < 2e-2
    # (2) linearity in V (bf16 rounding of the summed V and of the outputs only)
    assert (o12 - (o1 + o2)).abs().max().item() < 6e-2
    # (3) constant V -> constant output (softmax rows sum to one)
    oc = run(torch.full_like(v1, 0.5))
    assert (oc - 0.5).abs().max().item() < 4e-3
    assert int(pairs[1]) == int(((td[1][:, None] >= td[1][None, :])).sum())
