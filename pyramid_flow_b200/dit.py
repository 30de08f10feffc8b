"""B200FluxTransformer — drop-in for the reference `PyramidFluxTransformer` on the sampler hot path.

Mirrors the call surface `PyramidDiTForVideoGeneration` uses (pyramid_dit/pyramid_dit_for_video_gen_pipeline.py:760-766):

    dit(sample=[clips], timestep_ratio=t, encoder_hidden_states=e, encoder_attention_mask=m, pooled_projections=p)[0]

plus `.config.in_channels`, `.parameters()`, `.device`, `.dtype`, `.to()`; weights are imported from a state-dict in the
reference key layout.  The forward is a fixed sequence of libpf_b200 kernel launches on the current CUDA
stream (no torch math on the path, no CPU fallback):

  conditioning GEMVs -> all-layer AdaLN modulation GEMV -> embedders (GEMM, fp32 store into the joint residual stream)
  8 x double block : LN+modulate pre-pass | QKV GEMM (+bias, RMSNorm, RoPE epilogue) | masked joint attention |
                     out-proj GEMM (+gate*x+residual) | LN+modulate | FF1 GEMM (+GELU) | FF2 GEMM (+gate, residual)
  16 x single block: LN+modulate | QKV GEMM (+RMSNorm, RoPE) | proj_mlp GEMM (+GELU) | attention | proj_out GEMM over [attn|mlp]
  head             : LN+modulate (last-frame tokens only) | proj_out GEMM | unpatchify

gemm_precision="fp8" (opt-in, changes the numerics; include/pf_b200.h FP8 contract): the video-range QKV, to_out, FF1 and FF2
GEMMs of the double blocks and all three GEMMs of every single block run on e4m3 operands (per-token activation scales,
per-output-channel weight scales quantised once at import).  Their A operands come from the quantising LN-modulate or from
a row quantiser pass over `cat` (timer tag "quantize_fp8").  The text stream of the double blocks, the embedders, the head
and the conditioning / AdaLN GEMVs stay bf16.

The plan cache, workspace (its layout in HBM is described in joint_step.py), parallel layout and the launches the two
DiT drop-ins share live in joint_step.py; this module keeps miniFLUX's weight import, position ids and 3-axis RoPE, the
single-stream blocks, head padding under sequence parallelism and the NCCL formulation of the exchanges.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from . import ops, sp as SP
from ._lib import PF_EPI_GATE_RESID, PF_EPI_GELU_BF16
from .joint_step import DEFAULT_EXCHANGE, JointStep, StepLaunches, _Cfg, fp8_weight  # noqa: F401 (DEFAULT_EXCHANGE: bench.py)


@dataclass
class FluxConfigB200:
    """Same fields as the reference model's `config` (modeling_pyramid_flux.py:80-96)."""
    num_layers: int = 8
    num_single_layers: int = 16
    num_attention_heads: int = 30
    attention_head_dim: int = 64
    in_channels: int = 64
    joint_attention_dim: int = 4096
    pooled_projection_dim: int = 768
    axes_dims_rope: Tuple[int, ...] = (16, 24, 24)
    patch_size: int = 2

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim


# ----------------------------------------------------------------------------------------------------------------------
# host-side sequence plan: ids, RoPE table, segment/time ids, attention tile schedule (cached per shape+mask)
# ----------------------------------------------------------------------------------------------------------------------
def _axis_positions(n: int, n_fine: int) -> torch.Tensor:
    """Spatial positions of an n-wide clip on the finest clip's grid (reference: F.interpolate(arange, mode='linear'),
    modeling_pyramid_flux.py:193-204)."""
    if n == n_fine:
        return torch.arange(n_fine, dtype=torch.float32)
    return F.interpolate(torch.arange(n_fine, dtype=torch.float32)[None, None], n, mode="linear")[0, 0]


def build_position_ids(clip_thw: Sequence[Tuple[int, int, int]], text_len: int) -> torch.Tensor:
    """[S, 3] (time, y, x) ids for [text ; clips]; clip_thw are TOKEN grids (t, h/2, w/2) low-res -> high-res."""
    hf, wf = clip_thw[-1][1], clip_thw[-1][2]
    parts = [torch.zeros(text_len, 3)]
    t0 = 0
    for (t, h, w) in clip_thw:
        ids = torch.zeros(t, h, w, 3)
        ids[..., 0] = torch.arange(t0, t0 + t, dtype=torch.float32)[:, None, None]
        ids[..., 1] = _axis_positions(h, hf)[None, :, None]
        ids[..., 2] = _axis_positions(w, wf)[None, None, :]
        parts.append(ids.reshape(-1, 3))
        t0 += t
    return torch.cat(parts, 0)


def build_rope_table(ids: torch.Tensor, axes_dim: Sequence[int], theta: float = 10000.0) -> torch.Tensor:
    """(cos, sin) per rotation pair, [S, sum(axes)/2, 2] fp32, angles in fp64 (reference rope(), F:28-41)."""
    cols = []
    for i, d in enumerate(axes_dim):
        omega = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.float64) / d))
        ang = ids[:, i].to(torch.float64)[:, None] * omega[None]
        cols.append(torch.stack([ang.cos(), ang.sin()], -1))
    return torch.cat(cols, 1).to(torch.float32).contiguous()


@dataclass
class SeqPlan:
    text_len: int
    video_len: int
    seq: int
    last_tokens: int          # tokens of the current (last) clip
    clip_thw: Tuple[Tuple[int, int, int], ...]
    rope: torch.Tensor        # device fp32 [S, sum(axes_dim)/2, 2]
    seg: torch.Tensor         # device int32 [B, S]
    time: torch.Tensor        # device int32 [B, S]
    sched: torch.Tensor       # device int32 [B, q_tiles, stride]
    sched2: object            # ops.PairSchedule on the device: pair schedule + row masks (pf_attn_build_pair_*)
    allowed_pairs: int        # sum over batch of allowed (q, kv) pairs (attention FLOP accounting)
    pos: Optional[torch.Tensor] = None   # SD3 MMDiT: device fp32 [video_len, D] positional table of the clip tokens


def build_seq_plan(clip_shapes: Sequence[Sequence[int]], mask_cpu: torch.Tensor, axes_dim, patch: int, device) -> SeqPlan:
    """ids, RoPE table over the id axes (axes_dim: rotary dims of each of (time, y, x), leading axes only if shorter),
    segment / time ids and the attention tile schedules of one (clip shapes, text mask)."""
    b, text_len = mask_cpu.shape
    clip_thw = tuple((int(s[-3]), int(s[-2]) // patch, int(s[-1]) // patch) for s in clip_shapes)
    ids = build_position_ids(clip_thw, text_len)
    video_len = sum(t * h * w for t, h, w in clip_thw)
    seq = text_len + video_len
    rope = build_rope_table(ids, axes_dim)
    # segment id: sample index + 1 for valid tokens, 0 for padded text (reference F:318-330)
    seg = torch.arange(1, b + 1, dtype=torch.int32)[:, None].repeat(1, seq)
    seg[:, :text_len][mask_cpu == 0] = 0
    time = ids[:, 0].to(torch.int32)[None].repeat(b, 1).contiguous()
    sched, pairs = ops.attn_build_schedule(seg, time)
    sched2 = ops.attn_build_pair_schedule(sched, seq, seg, time)
    t, h, w = clip_thw[-1]
    return SeqPlan(text_len, video_len, seq, t * h * w, clip_thw, rope.to(device), seg.to(device), time.to(device),
                   sched.to(device), sched2.to(device), int(pairs.sum()))


class B200FluxTransformer(JointStep):
    """Holder of packed bf16 weights + the kernel-launch sequence of one DiT step."""

    def __init__(self, config: FluxConfigB200, state_dict: Dict[str, torch.Tensor], device="cuda",
                 emulate_bf16_rounding: bool = False, gemm_precision: str = "bf16"):
        super().__init__(config, gemm_precision)
        # True reproduces the reference's bf16 rounding of the sinusoidal projection (E:195); False keeps fp32
        self.emulate_bf16_rounding = emulate_bf16_rounding
        self.config = _Cfg(in_channels=config.in_channels, num_layers=config.num_layers,
                           num_single_layers=config.num_single_layers,
                           num_attention_heads=config.num_attention_heads,
                           attention_head_dim=config.attention_head_dim,
                           joint_attention_dim=config.joint_attention_dim,
                           pooled_projection_dim=config.pooled_projection_dim)
        self.token_dim = config.in_channels      # the packed latent channels of one 2x2 patch
        self._import_state_dict(state_dict, torch.device(device))
        self.trim_last_block = True     # last single block on the current clip's rows only (exact; see _forward_eager)

    @classmethod
    def from_reference(cls, ref_module, device="cuda", **kw) -> "B200FluxTransformer":
        """Build from a loaded reference `PyramidFluxTransformer` (its `.config` + `.state_dict()`)."""
        rc = ref_module.config
        cfg = FluxConfigB200(num_layers=rc.num_layers, num_single_layers=rc.num_single_layers,
                             num_attention_heads=rc.num_attention_heads, attention_head_dim=rc.attention_head_dim,
                             in_channels=rc.in_channels, joint_attention_dim=rc.joint_attention_dim,
                             pooled_projection_dim=rc.pooled_projection_dim,
                             axes_dims_rope=tuple(rc.axes_dims_rope))
        return cls(cfg, ref_module.state_dict(), device=device, **kw)

    # -- weight import (reference key layout) ---------------------------------------------------------------------------
    def _import_state_dict(self, sd: Dict[str, torch.Tensor], device) -> None:
        c = self.cfg
        d = c.inner_dim

        def W(*names):  # concatenated bf16 weight [sum(out), in]
            return torch.cat([sd[n + ".weight"].float() for n in names], 0).to(device=device, dtype=torch.bfloat16).contiguous()

        def Bv(*names):
            return torch.cat([sd[n + ".bias"].float() for n in names], 0).to(device=device, dtype=torch.float32).contiguous()

        def V(name):
            return sd[name].float().to(device).contiguous()

        fp8 = self.gemm_precision == "fp8"

        def WQ(blk, key, *names):   # the weight of a GEMM that runs in fp8 under gemm_precision="fp8"
            if fp8:
                blk[key], blk["s" + key[1:]] = fp8_weight(sd, names, device)
            else:
                blk[key] = W(*names)

        reg = self.register_buffer
        reg("w_t1", W("time_text_embed.timestep_embedder.linear_1")); reg("b_t1", Bv("time_text_embed.timestep_embedder.linear_1"))
        reg("w_t2", W("time_text_embed.timestep_embedder.linear_2")); reg("b_t2", Bv("time_text_embed.timestep_embedder.linear_2"))
        reg("w_p1", W("time_text_embed.text_embedder.linear_1")); reg("b_p1", Bv("time_text_embed.text_embedder.linear_1"))
        reg("w_p2", W("time_text_embed.text_embedder.linear_2")); reg("b_p2", Bv("time_text_embed.text_embedder.linear_2"))
        reg("w_ctx", W("context_embedder")); reg("b_ctx", Bv("context_embedder"))
        reg("w_x", W("x_embedder")); reg("b_x", Bv("x_embedder"))
        reg("w_out", W("proj_out")); reg("b_out", Bv("proj_out"))

        # every AdaLN linear of the model, stacked: one GEMV per step
        mod_names, self.mod_off = [], {}
        off = 0
        for i in range(c.num_layers):
            for nm, k in ((f"transformer_blocks.{i}.norm1", 6), (f"transformer_blocks.{i}.norm1_context", 6)):
                mod_names.append(nm + ".linear"); self.mod_off[nm] = off; off += k * d
        for i in range(c.num_single_layers):
            nm = f"single_transformer_blocks.{i}.norm"
            mod_names.append(nm + ".linear"); self.mod_off[nm] = off; off += 3 * d
        mod_names.append("norm_out.linear"); self.mod_off["norm_out"] = off; off += 2 * d
        self.n_mod = off
        reg("w_mod", W(*mod_names)); reg("b_mod", Bv(*mod_names))

        self.dbl, self.sgl = [], []
        for i in range(c.num_layers):
            p = f"transformer_blocks.{i}"
            blk = dict(
                b_qkv=Bv(p + ".attn.to_q", p + ".attn.to_k", p + ".attn.to_v"),
                w_cqkv=W(p + ".attn.add_q_proj", p + ".attn.add_k_proj", p + ".attn.add_v_proj"),
                b_cqkv=Bv(p + ".attn.add_q_proj", p + ".attn.add_k_proj", p + ".attn.add_v_proj"),
                nq=V(p + ".attn.norm_q.weight"), nk=V(p + ".attn.norm_k.weight"),
                cnq=V(p + ".attn.norm_added_q.weight"), cnk=V(p + ".attn.norm_added_k.weight"),
                b_o=Bv(p + ".attn.to_out.0"),
                w_co=W(p + ".attn.to_add_out"), b_co=Bv(p + ".attn.to_add_out"),
                b_f1=Bv(p + ".ff.net.0.proj"),
                b_f2=Bv(p + ".ff.net.2"),
                w_cf1=W(p + ".ff_context.net.0.proj"), b_cf1=Bv(p + ".ff_context.net.0.proj"),
                w_cf2=W(p + ".ff_context.net.2"), b_cf2=Bv(p + ".ff_context.net.2"),
            )
            WQ(blk, "w_qkv", p + ".attn.to_q", p + ".attn.to_k", p + ".attn.to_v")
            WQ(blk, "w_o", p + ".attn.to_out.0")
            WQ(blk, "w_f1", p + ".ff.net.0.proj")
            WQ(blk, "w_f2", p + ".ff.net.2")
            for k2, v2 in blk.items():
                reg(f"dbl{i}_{k2}", v2)
            self.dbl.append(blk)
        for i in range(c.num_single_layers):
            p = f"single_transformer_blocks.{i}"
            blk = dict(
                b_qkv=Bv(p + ".attn.to_q", p + ".attn.to_k", p + ".attn.to_v"),
                b_mlp=Bv(p + ".proj_mlp"),
                nq=V(p + ".attn.norm_q.weight"), nk=V(p + ".attn.norm_k.weight"),
                b_out=Bv(p + ".proj_out"),
            )
            WQ(blk, "w_qkv", p + ".attn.to_q", p + ".attn.to_k", p + ".attn.to_v")
            WQ(blk, "w_mlp", p + ".proj_mlp")
            WQ(blk, "w_out", p + ".proj_out")
            for k2, v2 in blk.items():
                reg(f"sgl{i}_{k2}", v2)
            self.sgl.append(blk)

    def _build_plan(self, clip_shapes, mask_cpu: torch.Tensor) -> SeqPlan:
        return build_seq_plan(clip_shapes, mask_cpu, self.cfg.axes_dims_rope, self.cfg.patch_size, self.device)

    def _pad_heads(self, hp: int) -> None:
        """Zero input columns for the padded heads in every GEMM that reads the attention output (sp.py)."""
        if hasattr(self, "_padded"):
            return
        d, pad = self.cfg.inner_dim, (hp - self.cfg.num_attention_heads) * 64

        def padk(w):   # [N, D (+rest)] -> [N, Hp*64 (+rest)]
            z = torch.zeros(w.shape[0], pad, device=w.device, dtype=w.dtype)
            return torch.cat([w[:, :d], z, w[:, d:]], dim=1).contiguous()

        for blk in self.dbl:
            blk["w_o_p"], blk["w_co_p"] = padk(blk["w_o"]), padk(blk["w_co"])
        for blk in self.sgl:
            blk["w_out_p"] = padk(blk["w_out"])
        self._padded = True

    def _graph_key_fields(self) -> tuple:
        return super()._graph_key_fields() + (bool(self.trim_last_block),)

    # -- the step ------------------------------------------------------------------------------------------------------
    def _forward_eager(self, clips, timestep_ratio=None, encoder_hidden_states=None, encoder_attention_mask=None,
                       pooled_projections=None):
        st = StepLaunches(self, clips, encoder_attention_mask)
        d, b, sl, h, xn, mod, nm, wa, ldc = st.d, st.b, st.sl, st.h, st.xn, st.mod, st.nm, st.wa, st.ldc
        cat, fp8, nsp, T = st.cat, st.fp8, st.nsp, self.timer
        st.condition(timestep_ratio, pooled_projections)
        st.embed(clips, encoder_hidden_states)
        s, n_last = st.plan.seq, st.plan.last_tokens
        nccl = st.par and st.px is None     # the all_to_all_single formulation of the exchanges

        def exchange_begin():
            if nccl and nsp > 1:
                return SP.heads_to_sequence_qkv_begin(st.q[0], st.k[0], st.v[0], self.layout)
            return None

        def attention(pending=None, q_row_begin=0):
            if not (nccl and nsp > 1):
                return st.attention(q_row_begin)
            # Ulysses exchange: all (padded) heads of my token chunk -> my head group over the whole sequence
            qf, kf, vf = SP.heads_to_sequence_qkv_end(pending if pending is not None else exchange_begin())
            of = st.ws.get("of")
            if of is None:   # attention output of my head group over the whole sequence
                of = st.ws["of"] = torch.empty(s, (st.hp // nsp) * 64, device=self.device, dtype=torch.bfloat16)
            st.attn(qf[None], kf[None], vf[None], of[None], q_row_begin)
            cat[0, :, :wa].copy_(SP.sequence_to_heads(of, self.layout))

        pad = st.hp != st.hn
        for i, w in enumerate(self.dbl):
            offs = (self.mod_off[f"transformer_blocks.{i}.norm1_context"], self.mod_off[f"transformer_blocks.{i}.norm1"])
            wq, bq, nq, nk = (w["w_cqkv"], w["w_qkv"]), (w["b_cqkv"], w["b_qkv"]), (w["cnq"], w["nq"]), (w["cnk"], w["nk"])
            for j in (0, 1):
                st.ln_rows(j, offs[j] + 0 * d, offs[j] + 1 * d)              # (shift_msa, scale_msa) N:173/191
                st.qkv_rows(j, w, wq[j], bq[j], nq[j], nk[j])
            attention()
            st.joint_tail(w, offs, st.ranges, (w["w_co_p"], w["w_o_p"]) if pad else (w["w_co"], w["w_o"]), (w["b_co"], w["b_o"]),
                          (w["w_cf1"], w["w_f1"]), (w["b_cf1"], w["b_f1"]), (w["w_cf2"], w["w_f2"]), (w["b_cf2"], w["b_f2"]))

        for i, w in enumerate(self.sgl):
            o = self.mod_off[f"single_transformer_blocks.{i}.norm"]
            # Last block: only the current clip's tokens are read afterwards (F:380), so its queries, MLP and projection
            # run on the rows from the 128-aligned start of the current clip; K/V still cover every token.  Same kernels
            # on fewer rows: the kept rows are bit-identical.  (Single-GPU layout; SP chunks stay uniform.)
            r0 = ((s - n_last) // 128) * 128 if (self.trim_last_block and not st.par and i == len(self.sgl) - 1) else 0
            if fp8:
                rows = dict(batches=b, rows_per_batch=sl, row_begin=r0, row_count=sl - r0)
                st.ln8(o, o + d, 0, sl)
                st.qkv8(w["w_qkv"], w["s_qkv"], w["b_qkv"], w["nq"], w["nk"], 0, sl)
                with T("gemm_single_mlp_gelu"):
                    ops.gemm_fp8(st.xa8, st.sx8, w["w_mlp"], w["s_mlp"], w["b_mlp"], PF_EPI_GELU_BF16, out=cat, ldo=ldc,
                                 out_col_begin=wa, **rows)
                attention(q_row_begin=r0)
                st.quant8(0, ldc, r0, sl - r0)
                with T("gemm_single_out"):
                    ops.gemm_fp8(st.xn8, st.sc8, w["w_out"], w["s_out"], w["b_out"], PF_EPI_GATE_RESID, out=h, ldo=d,
                                 gate=mod[:, o + 2 * d:], gate_batch_stride=nm, **rows)
                continue
            st.ln(o, o + d, 0, sl)                                                                 # (shift, scale) N:232
            # two launches sharing A: measured faster than the fused q|k|v|mlp GEMM (PF_EPI_QKV_GELU), whose 192-wide
            # tiles slow the MLP half down (1.81 ms fused vs 0.60 + 0.62 ms split at S=15488)
            st.qkv(w["w_qkv"], w["b_qkv"], w["nq"], w["nk"], 0, sl)
            pending = exchange_begin()       # SP: the q/k/v all-to-alls run under the proj_mlp GEMM
            with T("gemm_single_mlp_gelu"):
                ops.gemm(xn, w["w_mlp"], w["b_mlp"], PF_EPI_GELU_BF16, batches=b, rows_per_batch=sl, row_begin=r0,
                         row_count=sl - r0, out=cat, ldo=ldc, out_col_begin=wa)
            attention(pending, q_row_begin=r0)
            with T("gemm_single_out"):
                ops.gemm(cat, w["w_out_p"] if pad else w["w_out"], w["b_out"], PF_EPI_GATE_RESID, batches=b,
                         rows_per_batch=sl, row_begin=r0, row_count=sl - r0, out=h, ldo=d, gate=mod[:, o + 2 * d:],
                         gate_batch_stride=nm)

        if not nccl:
            return [st.publish(st.unpatchify(st.head(), clips))]
        if nsp > 1:
            st.ws["head"].zero_()
        head = st.head()
        if nsp > 1:
            torch.distributed.all_reduce(head, group=self.layout.sp_group)       # disjoint row blocks: sum == gather
        out = st.unpatchify(head, clips)
        full = torch.empty(st.bg, *out.shape[1:], device=self.device, dtype=out.dtype)
        torch.distributed.all_gather_into_tensor(full, out, group=self.layout.cfg_group)   # [uncond ; cond]
        return [full]

    # accounting used by bench.py / DESIGN.md (algorithmic work per unit)
    def step_flops(self, b: int, plan: SeqPlan) -> Dict[str, float]:
        c = self.cfg
        d = c.inner_dim
        per_tok = 24.0 * d * d
        gemm = b * plan.seq * per_tok * (c.num_layers + c.num_single_layers)
        gemm += 2.0 * b * (plan.video_len * c.in_channels * d + plan.text_len * c.joint_attention_dim * d +
                           plan.last_tokens * d * c.in_channels)
        attn = 4.0 * 64 * c.num_attention_heads * plan.allowed_pairs * (c.num_layers + c.num_single_layers)
        return {"gemm": gemm, "attention": attn}
