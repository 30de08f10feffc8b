"""The varlen (flash path) training attention on the H100: the pack / unpack kernels bit for bit against the reference's torch
glue and autograd through it, varlen_attention against fp32 autograd per sequence (and flash_attn when it imports), and a
training step of the unmodified reference miniFLUX built with use_flash_attn=True."""
import copy
import sys

import pytest
import torch
import torch.nn.functional as F

from pyramid_flow_b200 import training

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _reference_block():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    return __import__("pyramid_dit.flux_modules.modeling_flux_block", fromlist=["apply_rope"]), ref_shim


# ---- torch stand-ins for the flash_attn helpers the reference calls (flash_attn.bert_padding semantics) ----------------
def index_first_axis(x, indices):
    return x[indices]


def pad_input(x, indices, batch, seqlen):
    out = torch.zeros(batch * seqlen, *x.shape[1:], dtype=x.dtype, device=x.device)
    out[indices] = x
    return out.view(batch, seqlen, *x.shape[1:])


def flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dropout_p=0.0, softmax_scale=None,
                           causal=False):
    """Non-causal attention within each sequence, one SDPA call per sequence, in the inputs' dtype."""
    assert dropout_p == 0.0 and not causal and torch.equal(cu_seqlens_q, cu_seqlens_k)
    cu = cu_seqlens_q.tolist()
    outs = []
    for a, b in zip(cu[:-1], cu[1:]):
        qi, ki, vi = (t[a:b].transpose(0, 1)[None] for t in (q, k, v))
        outs.append(F.scaled_dot_product_attention(qi, ki, vi, scale=softmax_scale)[0].transpose(0, 1))
    return torch.cat(outs)


def _freqs(g, b, seq):
    """[B, S, 1, 32, 2, 2] fp32 rotation tables of random positions, as EmbedND builds them."""
    pos = torch.randint(0, 64, (b, seq), generator=g).double()
    omega = 1.0 / (10000 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    ang = pos[..., None] * omega
    tab = torch.stack([ang.cos(), -ang.sin(), ang.sin(), ang.cos()], dim=-1).view(b, seq, 32, 2, 2)
    return tab.float().unsqueeze(2).to(DEV)


def _masks(b, n, text, valid):
    mask = torch.zeros(b * n, text, dtype=torch.long)
    for r in range(b * n):
        mask[r, :valid[r % len(valid)]] = 1
    return mask


def _stage_indices(mask, hidden_length, text_len):
    """merge_input's flash branch (F:295-317): per stage the indices / seqlens_in_batch of cat(text mask, ones)."""
    n = len(hidden_length)
    out = []
    for i_p, length in enumerate(hidden_length):
        m = mask[i_p::n]
        if text_len:
            m = torch.cat([m, torch.ones(m.shape[0], length, dtype=m.dtype)], dim=1)
        out.append({"indices": torch.nonzero(m.flatten()).flatten().to(DEV), "seqlens_in_batch": m.sum(-1, dtype=torch.int32).to(DEV)})
    return out


def _glue(video, text, freqs, hidden_length, stages, rope):
    """The reference's torch code before flash_attn_varlen_func (B:208-226, B:468-483), then the kernels' head-major bf16."""
    qkv = torch.stack(video, dim=2)
    enc = torch.stack(text, dim=2) if text is not None else None
    n, i_sum, parts = len(hidden_length), 0, []
    for i_p, length in enumerate(hidden_length):
        tokens = qkv[:, i_sum:i_sum + length]
        if enc is not None:
            tokens = torch.cat([enc[i_p::n], tokens], dim=1)
        if freqs is not None:
            tokens[:, :, 0], tokens[:, :, 1] = rope(tokens[:, :, 0], tokens[:, :, 1], freqs[i_p])
        parts.append(index_first_axis(tokens.flatten(0, 1), stages[i_p]["indices"]))
        i_sum += length
    return [t.transpose(0, 1).unsqueeze(0).contiguous().to(torch.bfloat16) for t in torch.cat(parts).unbind(1)]


def _glue_unpack(out, query_like, enc_like, hidden_length, stages, text_len):
    """B:247-262 / B:504-516: pad_input of each stage's rows into zeros_like(query) / zeros_like(encoder_query)."""
    b, _, h, hd = query_like.shape
    out = out.view(-1, h, hd)
    hidden = torch.zeros_like(query_like)
    encoder = torch.zeros_like(enc_like) if enc_like is not None else None
    n, i_sum, tok = len(hidden_length), 0, 0
    for i_p, length in enumerate(hidden_length):
        cnt = stages[i_p]["indices"].numel()
        st = pad_input(out[tok:tok + cnt], stages[i_p]["indices"], b, text_len + length)
        hidden[:, i_sum:i_sum + length] = st[:, text_len:]
        if encoder is not None:
            encoder[i_p::n] = st[:, :text_len]
        tok += cnt
        i_sum += length
    return hidden.flatten(2, 3), (encoder.flatten(2, 3) if encoder is not None else None)


_DTYPES = {"bf16": (torch.bfloat16,) * 3, "fp32": (torch.float32,) * 3, "mixed": (torch.float32, torch.float32, torch.bfloat16)}

PACK_CASES = {
    # name: batch, heads, text rows, valid text rows per encoder row, stage lengths, rope, source dtypes, joint form
    "joint3_bf16_rope": (2, 3, 128, [128, 1, 77, 40, 128, 5], [64, 190, 300], True, "bf16", True),
    "joint2_fp32_rope": (3, 2, 24, [24, 1, 7], [33, 100], True, "fp32", True),
    "joint3_mixed_norope": (2, 24, 40, [13, 40, 1], [40, 96, 257], False, "mixed", True),
    "single3_bf16_rope": (2, 3, 128, [128, 1, 64], [64, 190, 300], True, "bf16", False),
    "single2_fp32_rope": (3, 2, 24, [1, 24, 11], [33, 100], True, "fp32", False),
}


@pytest.mark.parametrize("case", list(PACK_CASES))
def test_pack_and_unpack_match_the_reference_glue(case):
    block, _ = _reference_block()
    b, h, text_len, valid, hidden_length, use_rope, dts, joint = PACK_CASES[case]
    dtypes = _DTYPES[dts]
    g = torch.Generator().manual_seed(len(case) + b)
    n = len(hidden_length)
    mask = _masks(b, n, text_len, valid)
    stage_len = [text_len + L for L in hidden_length]
    stages = _stage_indices(mask, hidden_length, text_len)
    plan = training.varlen_plan([s["indices"] for s in stages], [s["seqlens_in_batch"] for s in stages], b, stage_len)
    if joint:
        video = [torch.randn(b, sum(hidden_length), h, 64, generator=g).to(DEV, dt).requires_grad_() for dt in dtypes]
        text = [torch.randn(b * n, text_len, h, 64, generator=g).to(DEV, dt).requires_grad_() for dt in dtypes]
        seq_lens, stage_row0, src_text, glue_text_len = hidden_length, [sum(hidden_length[:i]) for i in range(n)], text, text_len
    else:   # the single blocks: each stage's text rows are already part of the stage-major sequence
        video = [torch.randn(b, sum(stage_len), h, 64, generator=g).to(DEV, dt).requires_grad_() for dt in dtypes]
        text = None
        seq_lens, stage_row0, src_text, glue_text_len = stage_len, [sum(stage_len[:i]) for i in range(n)], None, 0
    freqs = [_freqs(g, b, s) for s in stage_len] if use_rope else None
    leaves = video + (text or [])

    # pack: q / k / v against the glue, source gradients against autograd through it
    grads = [torch.randn(1, h, plan.total, 64, generator=g).to(DEV, torch.bfloat16) for _ in range(3)]
    packed = training._VarlenPack.apply(plan, stage_row0, text is not None, *video, *(text or []), *(freqs or []))
    torch.autograd.backward(packed, grads)
    ours = [t.grad.clone() for t in leaves]
    for t in leaves:
        t.grad = None
    want = _glue(video, src_text, freqs, seq_lens, stages, block.apply_rope)
    torch.autograd.backward(want, grads)
    for i, (p, w) in enumerate(zip(packed, want)):
        assert p.shape == w.shape and torch.equal(p, w), f"{case}: packed {'qkv'[i]} differs"
    for i, (o, t) in enumerate(zip(ours, leaves)):
        assert o.dtype == t.dtype and torch.equal(o, t.grad), f"{case}: gradient of source {i} differs"
    if text is not None:       # the dropped (padded) text rows get a gradient of exactly 0
        dropped = (mask == 0).to(DEV)
        for o in ours[3:]:
            assert not bool(o[dropped].any())

    # unpack: the scatter into zeros, and the gather of its gradients (a strided view of a wider gradient, as B:936 gives)
    out = torch.randn(1, plan.total, h * 64, generator=g).to(DEV, torch.bfloat16).requires_grad_()
    mlp = torch.randn(b, video[0].shape[1], 96, generator=g).to(DEV, dtypes[0])
    w_video = torch.randn(b, video[0].shape[1], h * 64 + 96, generator=g).to(DEV)
    w_text = torch.randn(b * n, text_len, h * 64, generator=g).to(DEV) if text is not None else None

    def loss(res):
        vid, enc = res if text is not None else (res, None)
        total = (torch.cat([vid, mlp.to(vid.dtype)], dim=2).float() * w_video).sum()
        return total + ((enc.float() * w_text).sum() if enc is not None else 0), vid, enc

    l_ours, vid, enc = loss(training._VarlenUnpack.apply(plan, stage_row0, out, (b, video[0].shape[1], h * 64), video[0].dtype,
                                                         None if text is None else (b * n, text_len, h * 64),
                                                         None if text is None else text[0].dtype))
    l_ours.backward()
    g_ours = out.grad.clone()
    out.grad = None
    ref_vid, ref_enc = _glue_unpack(out, torch.zeros_like(video[0]), torch.zeros_like(text[0]) if text else None, seq_lens, stages,
                                    glue_text_len)
    l_ref, _, _ = loss((ref_vid, ref_enc) if text is not None else ref_vid)
    l_ref.backward()
    assert vid.dtype == video[0].dtype and torch.equal(vid, ref_vid)
    if text is not None:
        assert enc.dtype == text[0].dtype and torch.equal(enc, ref_enc)
        assert not bool(enc[(mask == 0).to(DEV)].any())
    assert torch.equal(g_ours, out.grad)


def _rel_rms(x, ref):
    return ((x.float() - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()


SEQLENS = {
    "short_in_one_tile": [5, 17, 1, 40, 31],               # several sequences inside one 128-row tile
    "ragged": [300, 77, 128, 1, 260, 9, 555],               # lengths not multiples of 128, boundaries inside tiles
    "one_long": [1000],
}


@pytest.mark.parametrize("case", list(SEQLENS))
def test_varlen_attention_against_fp32_per_sequence(case):
    lens = SEQLENS[case]
    g = torch.Generator().manual_seed(len(lens))
    total, h = sum(lens), 4
    q, k, v, dout = (torch.randn(total, h, 64, generator=g).to(DEV, torch.bfloat16) for _ in range(4))
    cu = F.pad(torch.cumsum(torch.tensor(lens), 0), (1, 0)).to(DEV, torch.int32)
    scale = 0.11

    def per_sequence(dtype):
        qs, ks, vs = (t.to(dtype).clone().requires_grad_() for t in (q, k, v))
        out = flash_attn_varlen_func(qs, ks, vs, cu, cu, max(lens), max(lens), softmax_scale=scale)
        out.backward(dout.to(dtype))
        return dict(out=out.detach().float(), dq=qs.grad.float(), dk=ks.grad.float(), dv=vs.grad.float())

    def ours(fn=training.varlen_attention):
        qs, ks, vs = (t.clone().requires_grad_() for t in (q, k, v))
        out = fn(qs, ks, vs, cu, softmax_scale=scale) if fn is training.varlen_attention else \
            fn(qs, ks, vs, cu, cu, max(lens), max(lens), softmax_scale=scale)
        out.backward(dout)
        return dict(out=out.detach(), dq=qs.grad, dk=ks.grad, dv=vs.grad)

    ref, sdpa = per_sequence(torch.float32), per_sequence(torch.bfloat16)
    first, second = ours(), ours()
    torch.cuda.synchronize()
    for name in ("out", "dq", "dk", "dv"):
        e_ours, e_sdpa = _rel_rms(first[name], ref[name]), _rel_rms(sdpa[name], ref[name])
        print(f"{case} {name}: relative RMS error vs fp32 {e_ours:.3e} (bf16 SDPA per sequence {e_sdpa:.3e})")
        assert first[name].dtype == torch.bfloat16 and first[name].shape == (total, h, 64)
        assert torch.isfinite(first[name]).all()
        assert e_ours <= 1.5 * e_sdpa, (case, name, e_ours, e_sdpa)
        assert torch.equal(first[name], second[name]), f"{case} {name}: two runs differ"
    try:
        from flash_attn import flash_attn_varlen_func as fa_varlen
    except ImportError:
        print("flash_attn does not import: the comparison with flash_attn_varlen_func is skipped")
        return
    fa = ours(fa_varlen)
    for name in ("out", "dq", "dk", "dv"):
        e_ours, e_fa = _rel_rms(first[name], ref[name]), _rel_rms(fa[name], ref[name])
        print(f"{case} {name}: flash_attn relative RMS error vs fp32 {e_fa:.3e}, ours {e_ours:.3e}")
        assert e_ours <= 1.5 * max(e_fa, e_sdpa)


# ---- a training step of the reference model on its flash path --------------------------------------------------------
def _flux():
    _, ref_shim = _reference_block()
    return __import__("pyramid_dit.flux_modules", fromlist=["PyramidFluxTransformer"]).PyramidFluxTransformer, ref_shim


def _model_inputs(bs=2):
    g = torch.Generator().manual_seed(17)
    # three stages of the no-AR pyramid: one clip per stage at rising resolution (t2v: two frames)
    sample = [[torch.randn(bs, 16, 2, 8, 16, generator=g)], [torch.randn(bs, 16, 2, 16, 32, generator=g)],
              [torch.randn(bs, 16, 2, 32, 64, generator=g)]]
    mask = _masks(bs, 3, 40, [40, 1, 13, 29, 7, 40])
    enc = torch.randn(3 * bs, 40, 64, generator=g)
    pooled = torch.randn(3 * bs, 32, generator=g)
    t = torch.tensor([900.0, 500.0, 100.0] * bs)
    targets = [torch.randn(*c[0].shape, generator=g) for c in sample]
    return sample, enc, mask, pooled, t, targets


def _train_step(model, inputs, dtype, autocast):
    sample, enc, mask, pooled, t, targets = inputs
    model.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        preds = model(sample=[[c.to(DEV, dtype) for c in clips] for clips in sample], encoder_hidden_states=enc.to(DEV, dtype),
                      encoder_attention_mask=mask.to(DEV), pooled_projections=pooled.to(DEV, dtype), timestep_ratio=t.to(DEV, dtype))
        loss = sum(((p.float() - y.to(DEV)) ** 2).mean() for p, y in zip(preds, targets))
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().float().clone() for n, p in model.named_parameters() if p.grad is not None}
    return loss.detach().float(), grads


def _compare(g_ours, g_ref, g32):
    assert set(g_ours) == set(g32) == set(g_ref) and len(g32) > 10
    num = lambda gs: torch.cat([(gs[n] - g32[n]).flatten() for n in g32]).pow(2).sum().sqrt().item()
    den = torch.cat([g32[n].flatten() for n in g32]).pow(2).sum().sqrt().item()
    return num(g_ours) / den, num(g_ref) / den


def _recording(model, mask):
    """Wraps the installed callables to check that dropped text rows get an output of exactly 0 and q / k / v gradients of
    exactly 0."""
    seen = {"out": 0, "grad": 0}
    n = 3
    dropped = (mask == 0).to(DEV)

    def check_grad(rows):
        def hook(grad):
            assert not bool(grad[rows].any())
            seen["grad"] += 1
        return hook

    for m in model.modules():
        proc = getattr(m, "processor", None)
        if type(proc).__name__ not in ("FluxAttnProcessor2_0", "FluxSingleAttnProcessor2_0"):
            continue
        inner = proc.varlen_flash_attn
        if type(proc).__name__ == "FluxAttnProcessor2_0":
            def joint(q, k, v, eq, ek, ev, *args, inner=inner):
                for t in (eq, ek, ev):
                    if t.requires_grad:
                        t.register_hook(check_grad(dropped))
                out, enc = inner(q, k, v, eq, ek, ev, *args)
                assert not bool(enc[dropped].any())
                seen["out"] += 1
                return out, enc
            proc.varlen_flash_attn = joint
        else:
            def single(q, k, v, heads, scale, hidden_length, *args, inner=inner):
                b = q.shape[0]
                rows = torch.cat([torch.cat([dropped[i::n], torch.zeros(b, L - dropped.shape[1], dtype=torch.bool, device=DEV)], 1)
                                  for i, L in enumerate(hidden_length)], dim=1)
                for t in (q, k, v):
                    if t.requires_grad:
                        t.register_hook(check_grad(rows))
                out = inner(q, k, v, heads, scale, hidden_length, *args)
                assert not bool(out[rows].any())
                seen["out"] += 1
                return out
            proc.varlen_flash_attn = single
    return seen


@pytest.mark.parametrize("param_dtype", [torch.float32, torch.bfloat16])
def test_reference_flash_training_step(param_dtype, monkeypatch):
    flux, ref_shim = _flux()
    block = sys.modules[flux.__module__.rsplit(".", 1)[0] + ".modeling_flux_block"]
    cfg = dict(num_layers=2, num_single_layers=2, num_attention_heads=3, attention_head_dim=64, in_channels=64,
               joint_attention_dim=64, pooled_projection_dim=32, use_flash_attn=True, use_gradient_checkpointing=True,
               gradient_checkpointing_ratio=1.0)
    model = flux(**cfg)
    ref_shim.reinit_all_parameters(model, seed=7, std=0.05)
    model32 = copy.deepcopy(model).to(DEV).train()
    model = model.to(DEV, param_dtype).train()
    inputs = _model_inputs()

    # the reference's own flash path with the torch stand-ins: in fp32, and in bf16 as the library path runs it
    monkeypatch.setattr(block, "flash_attn_varlen_func", flash_attn_varlen_func)
    monkeypatch.setattr(block, "index_first_axis", index_first_axis, raising=False)
    monkeypatch.setattr(block, "pad_input", pad_input, raising=False)
    loss32, g32 = _train_step(model32, inputs, torch.float32, autocast=False)
    loss_ref, g_ref = _train_step(model, inputs, param_dtype, autocast=True)

    def absent(*a, **k):
        raise AssertionError("the installed path called flash_attn_varlen_func")

    monkeypatch.setattr(block, "flash_attn_varlen_func", absent)
    training.install_varlen_training_attention(model)
    try:
        seen = _recording(model, inputs[2])
        loss_ours, g_ours = _train_step(model, inputs, param_dtype, autocast=True)
        loss_ours2, g_ours2 = _train_step(model, inputs, param_dtype, autocast=True)
    finally:
        training.uninstall_training_attention(model)
    assert seen["out"] >= 8 and seen["grad"] > 0

    e_ours, e_ref = _compare(g_ours, g_ref, g32)
    print(f"{param_dtype}: loss fp32 {loss32.item():.6f}, bf16 reference path {loss_ref.item():.6f}, installed "
          f"{loss_ours.item():.6f}; all gradients, relative error vs fp32: installed {e_ours:.3e}, reference bf16 {e_ref:.3e}")
    assert e_ours <= 1.5 * e_ref
    if param_dtype == torch.float32:
        for n in g32:
            d = g32[n].norm().item()
            if d == 0:
                continue
            eo, er = (g_ours[n] - g32[n]).norm().item() / d, (g_ref[n] - g32[n]).norm().item() / d
            assert eo <= 1.5 * max(er, 1e-3), (n, eo, er)
        assert abs(loss_ours - loss32) <= 1.5 * abs(loss_ref - loss32) + 1e-6 * abs(loss32)
    else:
        assert abs(loss_ours - loss32) <= 1.5 * abs(loss_ref - loss32) + 1e-3 * abs(loss32)
    assert torch.equal(loss_ours, loss_ours2) and all(torch.equal(g_ours[n], g_ours2[n]) for n in g_ours)
