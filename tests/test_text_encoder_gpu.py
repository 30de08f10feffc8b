"""Text encoders on the H100: each new kernel against fp32 PyTorch on the same bf16 inputs, both wrappers against the
reference wrappers' outputs (tests/golden/text_encoder_small.pt) through strings, the full-width encoders against the fp32
oracle, the drop-in from_reference, and the CPU offload round trip."""
import pytest
import torch
import torch.nn.functional as F

from oracle import text_encoder_oracle as TO

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-20)).item()


def _rel_rms(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


# ---- pf_attn_fwd_text -----------------------------------------------------------------------------------------------
def _attn_ref(qkv, batch, heads, seq, scale, bias, mask, causal):
    x = qkv.float().view(batch, seq, 3, heads, 64).permute(2, 0, 3, 1, 4)     # [3, B, H, S, 64]
    s = scale * x[0] @ x[1].transpose(-1, -2)
    if bias is not None:
        q = torch.arange(seq, device=DEV)[:, None]
        k = torch.arange(seq, device=DEV)[None, :]
        s = s + bias[:, k - q + seq - 1][None]
    allowed = torch.ones(batch, 1, seq, seq, dtype=torch.bool, device=DEV)
    if mask is not None:
        allowed &= mask.bool()[:, None, None, :]
    if causal:
        allowed &= torch.ones(seq, seq, dtype=torch.bool, device=DEV).tril()
    p = torch.softmax(s.masked_fill(~allowed, float("-inf")), dim=-1)
    return (p @ x[2]).transpose(1, 2).reshape(batch * seq, heads * 64)


@pytest.mark.parametrize("seq", [77, 128, 256])
@pytest.mark.parametrize("heads", [2, 12, 64])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("with_bias", [False, True])
def test_attn_text_matches_torch(seq, heads, causal, with_bias):
    from pyramid_flow_b200 import _lib, ops
    _lib.require_device()
    B = 2
    g = torch.Generator(device=DEV).manual_seed(seq * 131 + heads * 7 + 2 * causal + with_bias)
    # padded row strides on both sides (ld_qkv, ldo > the packed widths)
    qkv_buf = torch.randn(B * seq, 3 * heads * 64 + 64, device=DEV, generator=g).bfloat16()
    qkv = qkv_buf[:, :3 * heads * 64]
    out_buf = torch.zeros(B * seq, heads * 64 + 64, device=DEV, dtype=torch.bfloat16)
    out = out_buf[:, :heads * 64]
    bias = (torch.randn(heads, 2 * seq - 1, device=DEV, generator=g) * 2.0) if with_bias else None
    mask = (torch.rand(B, seq, device=DEV, generator=g) < 0.7).to(torch.int32)
    mask[:, 0] = 1                       # every row keeps a key (key 0 also passes the causal mask)
    mask[1, seq // 3:] = 0               # a ragged padded tail
    scale = 0.125 if causal else 0.5
    ops.attn_fwd_text(qkv, out, batch=B, heads=heads, seq=seq, scale=scale, bias=bias, key_mask=mask, causal=causal)
    torch.cuda.synchronize()
    ref = _attn_ref(qkv, B, heads, seq, scale, bias, mask, causal)
    assert (out.float() - ref).abs().max().item() < 2e-2
    assert bool((out_buf[:, heads * 64:] == 0).all())


def test_attn_text_without_mask():
    from pyramid_flow_b200 import _lib, ops
    _lib.require_device()
    B, H, S = 3, 4, 200
    g = torch.Generator(device=DEV).manual_seed(5)
    qkv = torch.randn(B * S, 3 * H * 64, device=DEV, generator=g).bfloat16()
    out = torch.empty(B * S, H * 64, device=DEV, dtype=torch.bfloat16)
    ops.attn_fwd_text(qkv, out, batch=B, heads=H, seq=S, scale=0.25)
    assert (out.float() - _attn_ref(qkv, B, H, S, 0.25, None, None, False)).abs().max().item() < 2e-2


# ---- GEMM epilogues -------------------------------------------------------------------------------------------------
def _epi_ref(name, y):
    if name == "geglu":
        m, n = y.shape
        t = y.view(m, n // 128, 2, 64)
        return (F.gelu(t[:, :, 0], approximate="tanh") * t[:, :, 1]).reshape(m, n // 2)
    if name == "quick":
        return y * torch.sigmoid(1.702 * y)
    return F.gelu(y)


def _epi_code(name):
    from pyramid_flow_b200 import _lib
    return {"geglu": _lib.PF_EPI_GEGLU_BF16, "quick": _lib.PF_EPI_QUICK_GELU_BF16, "erf": _lib.PF_EPI_GELU_ERF_BF16}[name]


@pytest.mark.parametrize("name", ["geglu", "quick", "erf"])
@pytest.mark.parametrize("M", [333, 8400])
def test_text_epilogues_match_torch_on_every_kernel(name, M):
    """Variant 1 = the 256 x 128 cluster kernel; variant 0 at M = 333 takes a 128-row kernel by the wave-tiling choice (128 x 64
    for quick / erf, 128 x 128 for GEGLU, which never takes 64-wide tiles), at M = 8400 the 128 x 128 kernel for quick / erf;
    variant 2 = the 128 x 64 kernel (quick / erf only).  Every kernel gives the same bits."""
    from pyramid_flow_b200 import _lib, ops
    _lib.require_device()
    K, N = 320, 512
    g = torch.Generator(device=DEV).manual_seed(M + len(name))
    x = (torch.randn(M, K, device=DEV, generator=g) * 0.5).bfloat16()
    w = (torch.randn(N, K, device=DEV, generator=g) * (1.5 / K ** 0.5)).bfloat16()
    bias = torch.randn(N, device=DEV, generator=g) * 0.1
    ref = _epi_ref(name, x.float() @ w.float().t() + bias)
    width = ref.shape[1]
    variants = [1, 0] if name == "geglu" else [1, 0, 2]
    outs = []
    for v in variants:
        buf = torch.zeros(M, width + 64, device=DEV, dtype=torch.bfloat16)
        ops.gemm(x, w, bias, _epi_code(name), rows_per_batch=M, out=buf, out_col_begin=64, kernel_variant=v)
        torch.cuda.synchronize()
        assert _rel(buf[:, 64:], ref) < 8e-3, v
        assert bool((buf[:, :64] == 0).all())
        outs.append(buf)
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_geglu_refuses_64_wide_tiles():
    from pyramid_flow_b200 import _lib, ops
    _lib.require_device()
    x = torch.zeros(128, 64, device=DEV, dtype=torch.bfloat16)
    w = torch.zeros(256, 64, device=DEV, dtype=torch.bfloat16)
    out = torch.zeros(128, 128, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="GEGLU"):
        ops.gemm(x, w, None, _lib.PF_EPI_GEGLU_BF16, rows_per_batch=128, out=out, kernel_variant=2)
    with pytest.raises(RuntimeError, match="GEGLU"):
        ops.gemm(x, w[:192], None, _lib.PF_EPI_GEGLU_BF16, rows_per_batch=128, out=out)


# ---- RMSNorm rows and the embedding lookup ------------------------------------------------------------------------------
def test_rms_norm_rows_matches_torch():
    from pyramid_flow_b200 import _lib, ops
    _lib.require_device()
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(2, 100, 4096, device=DEV, generator=g) * 3.0
    w = 1 + 0.1 * torch.randn(4096, device=DEV, generator=g)
    y = torch.zeros(2, 100, 4096, device=DEV, dtype=torch.bfloat16)
    ops.rms_norm_rows(x, y, w, batches=2, rows_per_batch=100, row_begin=7, row_count=90, eps=1e-6)
    ref = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6) * w
    assert _rel(y[:, 7:97], ref[:, 7:97]) < 8e-3
    assert bool((y[:, :7] == 0).all()) and bool((y[:, 97:] == 0).all())


def test_embed_tokens_matches_torch():
    from pyramid_flow_b200 import _lib, ops
    _lib.require_device()
    g = torch.Generator(device=DEV).manual_seed(4)
    table = torch.randn(1000, 768, device=DEV, generator=g).bfloat16()
    pos = torch.randn(77, 768, device=DEV, generator=g).bfloat16()
    ids = torch.randint(0, 1000, (3 * 77,), device=DEV, generator=g).to(torch.int32)
    out = torch.empty(3 * 77, 768, device=DEV)
    ops.embed_tokens(ids, table, out, rows_per_batch=77, pos_table=pos)
    rows = torch.arange(3 * 77, device=DEV) % 77
    assert torch.equal(out, table.float()[ids.long()] + pos.float()[rows])
    out2 = torch.empty(3 * 77, 768, device=DEV)
    ids[5], ids[9] = 1000, -3            # out of range: a zero row, nothing read outside the table
    ops.embed_tokens(ids, table, out2, rows_per_batch=77)
    ok = torch.ones(3 * 77, dtype=torch.bool, device=DEV)
    ok[5] = ok[9] = False
    assert torch.equal(out2[ok], table.float()[ids.long()[ok]])
    assert bool((out2[~ok] == 0).all())


# ---- wrappers against the reference wrappers' outputs ------------------------------------------------------------------
def _golden(golden_dir):
    g = torch.load(golden_dir / "text_encoder_small.pt", weights_only=False)
    cfgs = {k: (TO.ClipTextConfig if k.split("_")[1] == "clip" else TO.T5EncoderConfig)(**v) for k, v in g["configs"].items()}
    params = {k: (TO.synthetic_clip_params if isinstance(c, TO.ClipTextConfig) else TO.synthetic_t5_params)(c, g["seeds"][k])
              for k, c in cfgs.items()}
    return g, cfgs, params


def _small_wrappers(g, cfgs, params):
    from pyramid_flow_b200.text_encoder import B200CLIPText, B200FluxTextEncoder, B200SD3TextEncoder, B200T5Encoder
    tok = g["tokenizers"]

    def clip_tok():
        return TO.clip_tokenizer(tok["clip_vocab"], tok["clip_merges"])

    flux = B200FluxTextEncoder(clip_tok(), TO.t5_tokenizer(tok["t5_tokenizer_json"]),
                               B200CLIPText(cfgs["flux_clip"], params["flux_clip"], DEV),
                               B200T5Encoder(cfgs["flux_t5"], params["flux_t5"], DEV))
    sd3 = B200SD3TextEncoder(clip_tok(), clip_tok(), TO.t5_tokenizer(tok["t5_tokenizer_json"]),
                             B200CLIPText(cfgs["sd3_clip_l"], params["sd3_clip_l"], DEV),
                             B200CLIPText(cfgs["sd3_clip_g"], params["sd3_clip_g"], DEV),
                             B200T5Encoder(cfgs["sd3_t5"], params["sd3_t5"], DEV))
    return flux, sd3


def _bf16_oracle(g, cfgs, params, name):
    p16 = {k: TO.to_dtype(v, torch.bfloat16) for k, v in params.items()}
    with torch.no_grad():
        if name == "flux":
            pooled = TO.clip_text_forward(p16["flux_clip"], cfgs["flux_clip"], g["clip_ids"])[1]
            return TO.t5_encoder_forward(p16["flux_t5"], cfgs["flux_t5"], g["t5_ids"], g["t5_mask"]), pooled
        pooled = torch.cat([TO.clip_text_forward(p16[k], cfgs[k], g["clip_ids"])[2] for k in ("sd3_clip_l", "sd3_clip_g")], -1)
        return TO.t5_encoder_forward(p16["sd3_t5"], cfgs["sd3_t5"], g["t5_ids"], g["t5_mask"]), pooled


def test_wrappers_match_reference_golden(golden_dir):
    g, cfgs, params = _golden(golden_dir)
    flux, sd3 = _small_wrappers(g, cfgs, params)
    for name, enc, pooled_dim in (("flux", flux, 128), ("sd3", sd3, 256)):
        pe, am, pooled = enc(g["prompts"], DEV)
        ref = g[name]
        n = len(g["prompts"])
        assert pe.dtype == torch.bfloat16 and pe.shape == (n, 128, cfgs["flux_t5"].d_model) and pe.device.type == "cuda"
        assert am.dtype == torch.int64 and torch.equal(am.cpu(), ref["prompt_attention_mask"])
        assert pooled.dtype == torch.bfloat16 and pooled.shape == (n, pooled_dim)
        o_pe, o_pooled = _bf16_oracle(g, cfgs, params, name)
        for ours, bf16, want in ((pe, o_pe, ref["prompt_embeds"]), (pooled, o_pooled, ref["pooled_prompt_embeds"])):
            e, e16 = _rel_rms(ours.cpu(), want), _rel_rms(bf16, want)
            print(f"[text golden] {name} {tuple(want.shape)}: rel RMS {e:.3e} (bf16 oracle {e16:.3e})")
            assert e <= 1.5 * e16 and e < 2e-2


# ---- full-width encoders against the fp32 oracle ----------------------------------------------------------------------
def _ragged_inputs(B, vocab_t5, vocab_clip, g):
    t5_len = [128, 37]
    t5_ids = torch.zeros(B, 128, dtype=torch.long)
    t5_mask = torch.zeros(B, 128, dtype=torch.long)
    clip_ids = torch.full((B, 77), 49407, dtype=torch.long)
    for b in range(B):
        t5_ids[b, :t5_len[b]] = torch.randint(2, vocab_t5, (t5_len[b],), generator=g)
        t5_ids[b, t5_len[b] - 1] = 1
        t5_mask[b, :t5_len[b]] = 1
        n = [77, 20][b]
        clip_ids[b, 0] = 49406
        clip_ids[b, 1:n - 1] = torch.randint(0, 49406, (n - 2,), generator=g)
    return t5_ids, t5_mask, clip_ids


def test_full_width_encoders_against_fp32_oracle():
    """CLIP-L (pooler_output), CLIP-G (text_embeds) and T5-XXL at full depth, synthetic weights at the init scales, B = 2 with
    a padded T5 prompt: relative RMS of ours and of the bf16-weights oracle (the reference's bf16 numerics) against the
    fp32 oracle.  Ours must be within 1.5x of the bf16 oracle's error."""
    from pyramid_flow_b200.text_encoder import B200CLIPText, B200T5Encoder
    g = torch.Generator().manual_seed(0)
    t5_ids, t5_mask, clip_ids = _ragged_inputs(2, TO.T5_XXL.vocab_size, 49408, g)
    ids_d, mask_d, clip_d = t5_ids.to(DEV), t5_mask.to(DEV), clip_ids.to(DEV)
    report = {}
    for name, cfg in (("clip_l", TO.CLIP_L), ("clip_g", TO.CLIP_G)):
        p = TO.synthetic_clip_params(cfg, seed=1, device=DEV)
        with torch.no_grad():
            _, pooled32, emb32 = TO.clip_text_forward(p, cfg, clip_d)
            _, pooled16, emb16 = TO.clip_text_forward(TO.to_dtype(p, torch.bfloat16), cfg, clip_d)
        ours = B200CLIPText(cfg, p, DEV)(clip_ids)
        want, bf16 = (pooled32, pooled16) if cfg.projection_dim is None else (emb32, emb16)
        report[name + " pooled"] = (_rel_rms(ours, want), _rel_rms(bf16, want))
        del p, ours
    p = TO.synthetic_t5_params(TO.T5_XXL, seed=2, device=DEV)
    with torch.no_grad():
        want = TO.t5_encoder_forward(p, TO.T5_XXL, ids_d, mask_d)
        bf16 = TO.t5_encoder_forward(TO.to_dtype(p, torch.bfloat16), TO.T5_XXL, ids_d, mask_d)
    enc = B200T5Encoder(TO.T5_XXL, p, DEV)
    del p
    ours = enc(t5_ids, t5_mask)
    valid = mask_d.bool()
    report["t5 valid rows"] = (_rel_rms(ours[valid], want[valid]), _rel_rms(bf16[valid], want[valid]))
    report["t5 pad rows"] = (_rel_rms(ours[~valid], want[~valid]), _rel_rms(bf16[~valid], want[~valid]))
    for k, (e, e16) in report.items():
        print(f"[text full width] {k}: rel RMS ours {e:.3e}, bf16 oracle {e16:.3e}, ratio {e / e16:.2f}")
    for k, (e, e16) in report.items():
        assert e <= 1.5 * e16, k


# ---- drop-in and offload ----------------------------------------------------------------------------------------------
def test_from_reference_matches_reference_wrappers(golden_dir):
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("no staged reference checkout (oracle/_ref): build() stages it where the reference is readable")
    from oracle.pin import make_text_golden as MTG
    from transformers import PreTrainedModel
    from pyramid_flow_b200.text_encoder import B200FluxTextEncoder, B200SD3TextEncoder
    g, cfgs, params = _golden(golden_dir)
    flux_ref, sd3_ref = MTG.build_wrappers(g["tokenizers"], cfgs, params)
    prompts = ["a small dog under the blue sky", "photo of a red house " * 9]
    for ref, cls in ((flux_ref, B200FluxTextEncoder), (sd3_ref, B200SD3TextEncoder)):
        ours = cls.from_reference(ref, device=DEV)
        assert not any(isinstance(m, PreTrainedModel) for m in ours.modules())
        want = ref(prompts, "cpu")
        got = ours(prompts, DEV)
        assert torch.equal(got[1].cpu(), want[1])
        for a, b in ((got[0], want[0]), (got[2], want[2])):
            assert a.shape == b.shape and _rel_rms(a.cpu(), b) < 2e-2


def test_cpu_offload_round_trip_keeps_bits(golden_dir):
    g, cfgs, params = _golden(golden_dir)
    flux, _ = _small_wrappers(g, cfgs, params)
    first = flux(g["prompts"], DEV)
    flux.to("cpu")
    assert flux.device.type == "cpu"
    with pytest.raises(RuntimeError, match="no CPU path"):
        flux(g["prompts"], "cpu")
    flux.to("cuda")
    assert flux.device.type == "cuda" and flux.dtype == torch.bfloat16
    second = flux(g["prompts"], DEV)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
