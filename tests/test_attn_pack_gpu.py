"""The stage pack of the training attention (pf_attn_stage_pack / _bwd) against the torch code it replaces, bit for bit: the
stack of q / k / v, the cat of a stage's text rows with its video rows, the reference's fp32 apply_rope of both models,
transpose(1, 2).contiguous() and the cast to bf16; and autograd's gradients through that code."""
import ctypes as C

import pytest
import torch

from pyramid_flow_b200 import _lib, training

DEV = torch.device("cuda:0")


def _reference_ropes():
    from oracle.pin import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("the reference's sources are not staged (oracle/_ref)")
    ref_shim.install()
    flux = __import__("pyramid_dit.flux_modules.modeling_flux_block", fromlist=["apply_rope"])
    mmdit = __import__("pyramid_dit.mmdit_modules.modeling_mmdit_block", fromlist=["VarlenSelfAttentionWithT5Mask"])
    return {"flux": flux.apply_rope, "mmdit": mmdit.VarlenSelfAttentionWithT5Mask().apply_rope}


def _glue(video, text, freqs, hidden_length, rope):
    """The torch code of the drop-in before the pack kernels (and of the reference call sites up to SDPA): per stage the
    kernels' bf16 [B, H, T + L, 64] q, k, v."""
    qkv = torch.stack(video, dim=2)
    enc = torch.stack(text, dim=2) if text is not None else None
    n, i_sum, out = len(hidden_length), 0, []
    for i_p, length in enumerate(hidden_length):
        tokens = qkv[:, i_sum:i_sum + length]
        if enc is not None:
            tokens = torch.cat([enc[i_p::n], tokens], dim=1)
        q, k, v = tokens.unbind(2)
        if freqs is not None:
            q, k = rope(q, k, freqs[i_p])
        out += [t.transpose(1, 2).contiguous().to(torch.bfloat16) for t in (q, k, v)]
        i_sum += length
    return out


def _freqs(g, b, seq):
    """[B, S, 1, 32, 2, 2] fp32 rotation tables as the models' EmbedND / EmbedNDRoPE build them, from random positions."""
    pos = torch.randint(0, 64, (b, seq), generator=g).double()
    omega = 1.0 / (10000 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))
    ang = pos[..., None] * omega
    tab = torch.stack([ang.cos(), -ang.sin(), ang.sin(), ang.cos()], dim=-1).view(b, seq, 32, 2, 2)
    return tab.float().unsqueeze(2).to(DEV)


_DTYPES = {"bf16": (torch.bfloat16,) * 3, "fp32": (torch.float32,) * 3,
           # miniFLUX under bf16 autocast with fp32 parameters: its qk RMSNorm returns fp32 q / k, v is the Linear's bf16
           "mixed": (torch.float32, torch.float32, torch.bfloat16)}

CASES = {
    # name: batch, heads, text rows per stage (0 = the single blocks' form), stage lengths, rope, dtypes, fused qkv layout
    "joint1_bf16_rope": (1, 3, 77, [200], True, "bf16", False),
    "joint2_fp32_rope_fused": (3, 3, 13, [64, 190], True, "fp32", True),
    "joint3_mixed_rope": (3, 24, 129, [40, 96, 257], True, "mixed", False),
    "joint2_bf16_norope_fused": (1, 24, 24, [100, 300], False, "bf16", True),
    "joint3_fp32_norope": (3, 3, 7, [33, 65, 130], False, "fp32", False),
    "single2_mixed_rope": (3, 3, 0, [141, 267], True, "mixed", False),
    "single1_bf16_rope_fused": (1, 24, 0, [333], True, "bf16", True),
    "single3_bf16_norope": (3, 3, 0, [50, 77, 200], False, "bf16", False),
}


def _sources(g, b, h, rows, dtypes, fused):
    """Leaf tensors and the q / k / v views the models hand over: [B, S, H, 64] views of the Linear outputs (fused: of one
    [B, S, 3, H, 64] buffer, row stride 3 * H * 64, as a fused QKV projection gives)."""
    if fused:
        leaf = torch.randn(b, rows, 3, h, 64, generator=g).to(DEV, dtypes[0]).requires_grad_()
        return [leaf], [leaf[:, :, i] for i in range(3)]
    leaves = [torch.randn(b, rows, h * 64, generator=g).to(DEV, dt).requires_grad_() for dt in dtypes]
    return leaves, [t.view(b, rows, h, 64) for t in leaves]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_pack_and_its_gradients_match_the_torch_glue(case):
    b, h, text_len, hidden_length, use_rope, dts, fused = CASES[case]
    dtypes = _DTYPES[dts]
    ropes = _reference_ropes() if use_rope else {"none": None}
    g = torch.Generator().manual_seed(len(case) * 7 + b)
    n = len(hidden_length)
    vleaves, video = _sources(g, b, h, sum(hidden_length), dtypes, fused)
    tleaves, text = _sources(g, b * n, h, text_len, dtypes, fused) if text_len else ([], None)
    freqs = [_freqs(g, b, text_len + length) for length in hidden_length] if use_rope else None
    grads = [torch.randn(b, h, text_len + length, 64, generator=g).to(DEV, torch.bfloat16)
             for length in hidden_length for _ in range(3)]
    leaves = vleaves + tleaves

    srcs = tuple(video) + (tuple(text) if text is not None else ())
    packed = training._StagePack.apply(list(hidden_length), text is not None, *srcs, *(freqs or ()))
    torch.autograd.backward(packed, grads)
    ours = [t.grad.clone() for t in leaves]

    for name, rope in ropes.items():
        for t in leaves:
            t.grad = None
        want = _glue(video, text, freqs, hidden_length, rope)
        torch.autograd.backward(want, grads)
        for i, (p, w) in enumerate(zip(packed, want)):
            assert p.dtype == torch.bfloat16 and p.is_contiguous() and p.shape == w.shape
            assert torch.equal(p, w), f"{case} {name}: stage {i // 3} {'qkv'[i % 3]} differs"
        for i, (o, t) in enumerate(zip(ours, leaves)):
            assert o.dtype == t.dtype and torch.equal(o, t.grad), f"{case} {name}: gradient of source {i} differs"


def test_pack_rejects_bad_descriptors_without_a_launch():
    """Argument validation is host-side and happens before any CUDA call; pointers are dummies, never dereferenced."""
    from pyramid_flow_b200._lib import AttnPackDesc
    lib = _lib.load()
    dummy = 0x1000

    def desc():
        d = AttnPackDesc()
        d.batch, d.heads, d.head_dim, d.text_len, d.rows, d.row0, d.src_rows, d.n_stages, d.stage = 2, 3, 64, 24, 100, 50, 300, 2, 1
        for i in range(3):
            d.video[i] = d.text[i] = d.packed[i] = dummy
            for j, st in enumerate((300 * 192, 192, 64)):
                d.video_strides[i][j] = st
            for j, st in enumerate((24 * 192, 192, 64)):
                d.text_strides[i][j] = st
        return d

    launches = lib.pf_launch_count()
    bad = []
    d = desc(); d.head_dim = 128; bad.append((d, "head_dim"))
    d = desc(); d.row0 = 250; bad.append((d, "outside"))
    d = desc(); d.video_strides[1][1] = 196; bad.append((d, "multiple of 8"))
    d = desc(); d.text[2] = dummy + 8; bad.append((d, "aligned"))
    d = desc(); d.stage = 2; bad.append((d, "stage"))
    d = desc(); d.video_f32[0] = 2; bad.append((d, "fp32"))
    d = desc(); d.freqs, d.freqs_batch_stride, d.freqs_row_stride = dummy, 124 * 128, 64; bad.append((d, "freqs"))
    for d, what in bad:
        for entry in (lib.pf_attn_stage_pack, lib.pf_attn_stage_pack_bwd):
            assert entry(C.byref(d), None) < 0 and what in lib.pf_last_error().decode(), (what, lib.pf_last_error())
    assert lib.pf_attn_stage_pack(None, None) < 0 and "null" in lib.pf_last_error().decode()
    assert lib.pf_launch_count() == launches
