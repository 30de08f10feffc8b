"""The SD3 MMDiT with gemm_precision="fp8" on the GPU: the 24-block step against the fp32 oracle (the ragged-text 384p-like
pyramid of test_fulldepth_gpu.py and the full-size bench workload), CUDA-graph replay against host launches for both
precisions, and the default precision's bits."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# Regression tolerances on the relative RMS error of the velocity against the fp32 oracle: 1.3 x the value this
# implementation measured (the convention of test_fp8_gpu.py), on synthetic weights: a proxy for trained weights, not a
# quality figure.  Measured on an H100 80GB HBM3:
TOL_FP8_384P_REL_RMS = 1.3 * 3.13e-2    # S = 128 + 1320: measured 3.13e-2, cosine 0.99951 (the bf16 model: 2.10e-3)
TOL_FP8_FULL_REL_RMS = 1.3 * 3.10e-2    # S = 11888: measured 3.10e-2, cosine 0.99952 (the bf16 model: 2.15e-3)
MIN_FP8_COSINE = 0.99


def _stats(out, ref):
    d = out - ref
    return dict(max_abs=d.abs().max().item(), rel_rms=(d.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item(),
                cosine=F.cosine_similarity(out.flatten().double(), ref.flatten().double(), dim=0).item())


def _inputs_384p():
    """test_fulldepth_gpu.test_24_block_mmdit_step_matches_oracle's inputs: S = 128 + 1320, ragged text."""
    g = torch.Generator().manual_seed(22)
    clips = [torch.randn(2, 16, 2, 12, 20, generator=g), torch.randn(2, 16, 1, 24, 40, generator=g),
             torch.randn(2, 16, 1, 48, 80, generator=g)]
    clips = [c.bfloat16().float() for c in clips]
    enc = (torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().float()
    mask = torch.ones(2, 128, dtype=torch.long)
    mask[1, 61:] = 0
    pooled = torch.randn(2, 2048, generator=g)
    return dict(num_layers=24, pos_embed_max_size=96, sample_size=64), 21, clips, enc, mask, pooled, torch.tensor([640.0, 640.0])


def _inputs_full():
    """bench.py --model mmdit's workload: S = 128 + 13x240 + 960 + 2x3840 = 11888 (fp32 clips holding bf16 values, so the
    velocity is stored in fp32)."""
    g = torch.Generator().manual_seed(100)
    shapes = [(2, 16, 13, 24, 40), (2, 16, 1, 48, 80), (2, 16, 1, 96, 160), (2, 16, 1, 96, 160)]
    clips = [torch.randn(s, generator=g).bfloat16().float() for s in shapes]
    enc = (torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().float()
    mask = torch.ones(2, 128, dtype=torch.long)
    pooled = torch.randn(2, 2048, generator=g).bfloat16().float()
    return dict(num_layers=24), 11, clips, enc, mask, pooled, torch.tensor([3.0, 3.0])


@pytest.mark.parametrize("case,seq,head_chunk,tol", [("384p", 1448, 0, TOL_FP8_384P_REL_RMS),
                                                      ("full", 11888, 3, TOL_FP8_FULL_REL_RMS)])
def test_24_block_fp8_mmdit_step_against_the_oracle(case, seq, head_chunk, tol):
    from oracle import mmdit_oracle as MO
    from pyramid_flow_b200.mmdit import B200MMDiT, MMDiTConfigB200
    from tests.test_fulldepth_gpu import _oracle_on_gpu
    dev = torch.device("cuda:0")
    kw, seed, clips, enc, mask, pooled, t = (_inputs_384p if case == "384p" else _inputs_full)()
    cfg = MO.MMDiTConfig(**kw)
    params = MO.synthetic_mmdit_params(cfg, seed=seed)
    call = dict(sample=[[c.to(dev) for c in clips]], timestep_ratio=t.to(dev), encoder_hidden_states=enc.to(dev),
                encoder_attention_mask=mask.to(dev), pooled_projections=pooled.to(dev))
    outs = {}
    for prec in ("bf16", "fp8"):
        model = B200MMDiT(MMDiTConfigB200(**{k: v for k, v in kw.items() if k != "sample_size"}), params, device=dev,
                          gemm_precision=prec)
        o = model(**call)[0]
        assert o.dtype == torch.float32 and model.last_plan.seq == seq
        outs[prec] = o.cpu()
        del model
        torch.cuda.empty_cache()
    pd = {k: v.to(dev) for k, v in params.items()}
    del params
    ref = _oracle_on_gpu(lambda: MO.mmdit_forward(pd, cfg, [c.to(dev) for c in clips], t.to(dev), enc.to(dev), mask,
                                                  pooled.to(dev)).float().cpu(), head_chunk=head_chunk)
    del pd
    torch.cuda.empty_cache()
    st = {p: _stats(o, ref) for p, o in outs.items()}
    for p in ("bf16", "fp8"):
        print(f"MMDiT 24 blocks @ S={seq}, {p} GEMMs vs fp32 oracle: max_abs {st[p]['max_abs']:.3e} "
              f"rel_rms {st[p]['rel_rms']:.3e} cosine {st[p]['cosine']:.6f}")
    print(f"fp8 vs bf16 model: {_stats(outs['fp8'], outs['bf16'])} | |v| mean {ref.abs().mean():.3f}")
    assert ref.abs().mean().item() > 0.1
    assert bool(torch.isfinite(outs["fp8"]).all())
    assert st["fp8"]["cosine"] >= MIN_FP8_COSINE
    assert st["fp8"]["rel_rms"] <= tol


def _small_model_and_call(**kw):
    """A 3-block SD3-width MMDiT on the bench workload (S = 11888; the last block is context_pre_only)."""
    from bench import random_mmdit_state_dict
    from pyramid_flow_b200.mmdit import B200MMDiT, MMDiTConfigB200
    dev = torch.device("cuda:0")
    cfg = MMDiTConfigB200(num_layers=3)
    sd = random_mmdit_state_dict(cfg, dev, seed=0)
    g = torch.Generator().manual_seed(100)
    shapes = [(2, 16, 13, 24, 40), (2, 16, 1, 48, 80), (2, 16, 1, 96, 160), (2, 16, 1, 96, 160)]
    call = dict(sample=[[torch.randn(s, generator=g).bfloat16().to(dev) for s in shapes]],
                timestep_ratio=torch.tensor([3.0, 3.0]).bfloat16().to(dev),
                encoder_hidden_states=(torch.randn(2, 128, 4096, generator=g) * 0.2).bfloat16().to(dev),
                encoder_attention_mask=torch.ones(2, 128, dtype=torch.int64, device=dev),
                pooled_projections=torch.randn(2, 2048, generator=g).bfloat16().to(dev))
    return B200MMDiT(cfg, sd, device=dev, **kw), call


@pytest.mark.parametrize("prec", ["bf16", "fp8"])
def test_mmdit_graph_replay_equals_host_launch(prec):
    model, call = _small_model_and_call(gemm_precision=prec)
    e1 = model(**call)[0].clone()
    e2 = model(**call)[0].clone()
    model.use_cuda_graph = True
    g1 = model(**call)[0].clone()
    g2 = model(**call)[0].clone()
    torch.cuda.synchronize()
    assert model.graph_replays == 2 and len(model._graphs) == 1 and model.graph_launches_replayed > 0
    assert bool(torch.isfinite(e1.float()).all())
    assert torch.equal(e1, e2) and torch.equal(e1, g1) and torch.equal(g1, g2)


def test_mmdit_default_precision_is_bitwise_the_bf16_step():
    model, call = _small_model_and_call()
    want = model(**call)[0].clone()
    del model
    bf16, call = _small_model_and_call(gemm_precision="bf16")
    got = bf16(**call)[0]
    torch.cuda.synchronize()
    assert torch.equal(want, got)
