"""B200MMDiT — drop-in for the reference `PyramidDiffusionMMDiT` (SD3 variant) on the sampler hot path.

Same call surface as `B200FluxTransformer` (pipeline P:760-766); weights from the reference state-dict key layout
(`pos_embed.{pos_embed,proj}`, `attn.norm_add_q/k`, last block without `to_add_out` / `ff_context`).
Reuses the miniFLUX kernels unchanged — 24 double blocks at D=1536 / 24 heads — with three host-side differences:
  * patch embed = conv2d(k=2, s=2) (mmdit_modules/modeling_embedding.py:231) run as the patchify + GEMM pair with the conv
    weight re-ordered to the (p1 p2 c) feature order; the cropped / bilinearly down-sampled 2-D sincos table
    (ME:269-308, interp_condition_pos=True) is pre-placed in the residual stream and the GEMM accumulates onto it;
  * RoPE table = ONE 64-wide axis over the running frame index (modeling_pyramid_mmdit.py:116, 235-262, 301-305);
  * the last block is `context_pre_only`: AdaLayerNormContinuous (scale, shift) on the text stream, no text update after
    attention (modeling_mmdit_block.py:585-622, 659-660); q/k RMSNorm eps is 1e-5 (JointAttention default, MB:409).

gemm_precision="fp8" (opt-in, changes the numerics; include/pf_b200.h FP8 contract): the video-range QKV, to_out, FF1 and FF2
GEMMs of every joint block, the video stream of the context_pre_only last block included, run on e4m3 operands (per-token
activation scales, per-output-channel weight scales quantised once at import), as in dit.py.  The text stream (add_*_proj,
to_add_out, ff_context), the patch embed, the context embedder, the head and the conditioning / AdaLN GEMVs stay bf16.
The workspace gains `xn8` (e4m3 twin of `cat`, its first B*S*D bytes also holding the LN-modulate output), `sx8` and
`sc8` (row scales); see joint_step.py, which holds the step scaffolding and launches this model shares with dit.py.

use_cuda_graph = True captures each (plan, input shapes and dtypes, precision) once and replays it (graphs.GraphedStep).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import torch
import torch.nn.functional as F

from .dit import SeqPlan, build_seq_plan
from .joint_step import JointStep, StepLaunches, _Cfg, fp8_weight


@dataclass
class MMDiTConfigB200:
    num_layers: int = 24
    num_attention_heads: int = 24
    attention_head_dim: int = 64
    in_channels: int = 16
    patch_size: int = 2
    joint_attention_dim: int = 4096
    pooled_projection_dim: int = 2048
    pos_embed_max_size: int = 192

    @property
    def inner_dim(self) -> int:
        return self.num_attention_heads * self.attention_head_dim


class B200MMDiT(JointStep):
    norm_eps = 1e-5       # JointAttention's q/k RMSNorm default (MB:409)

    def __init__(self, config: MMDiTConfigB200, state_dict: Dict[str, torch.Tensor], device="cuda",
                 gemm_precision: str = "bf16"):
        super().__init__(config, gemm_precision)
        self.config = _Cfg(in_channels=config.in_channels, num_layers=config.num_layers,
                           num_attention_heads=config.num_attention_heads, attention_head_dim=config.attention_head_dim,
                           joint_attention_dim=config.joint_attention_dim,
                           pooled_projection_dim=config.pooled_projection_dim, patch_size=config.patch_size)
        assert config.patch_size == 2
        self.token_dim = 4 * config.in_channels     # (p1 p2 c) features of one 2x2 patch
        self._import_state_dict(state_dict, torch.device(device))

    @classmethod
    def from_reference(cls, ref_module, device="cuda", **kw) -> "B200MMDiT":
        rc = ref_module.config
        cfg = MMDiTConfigB200(num_layers=rc.num_layers, num_attention_heads=rc.num_attention_heads,
                              attention_head_dim=rc.attention_head_dim, in_channels=rc.in_channels,
                              patch_size=rc.patch_size, joint_attention_dim=rc.joint_attention_dim,
                              pooled_projection_dim=rc.pooled_projection_dim, pos_embed_max_size=rc.pos_embed_max_size)
        return cls(cfg, ref_module.state_dict(), device=device, **kw)

    def _import_state_dict(self, sd, device) -> None:
        c = self.cfg
        d = c.inner_dim

        def W(*names):
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
        for a, n in (("t1", "time_text_embed.timestep_embedder.linear_1"), ("t2", "time_text_embed.timestep_embedder.linear_2"),
                     ("p1", "time_text_embed.text_embedder.linear_1"), ("p2", "time_text_embed.text_embedder.linear_2"),
                     ("ctx", "context_embedder"), ("out", "proj_out")):
            reg("w_" + a, W(n)); reg("b_" + a, Bv(n))
        # conv2d weight [D, C, p1, p2] -> linear over patchified features ordered (p1 p2 c)
        wp = sd["pos_embed.proj.weight"].float().permute(0, 2, 3, 1).reshape(d, -1)
        reg("w_x", wp.to(device=device, dtype=torch.bfloat16).contiguous()); reg("b_x", V("pos_embed.proj.bias"))
        self.pos_table = sd["pos_embed.pos_embed"][0].float()        # [max*max, D] stays on the host; crops are cached per plan
        reg("ones_gate", torch.ones(1, d, device=device, dtype=torch.float32))

        mod_names, self.mod_off, off = [], {}, 0
        for i in range(c.num_layers):
            last = i == c.num_layers - 1
            for nm, k in ((f"transformer_blocks.{i}.norm1", 6), (f"transformer_blocks.{i}.norm1_context", 2 if last else 6)):
                mod_names.append(nm + ".linear"); self.mod_off[nm] = off; off += k * d
        mod_names.append("norm_out.linear"); self.mod_off["norm_out"] = off; off += 2 * d
        self.n_mod = off
        reg("w_mod", W(*mod_names)); reg("b_mod", Bv(*mod_names))

        self.blocks = []
        for i in range(c.num_layers):
            p = f"transformer_blocks.{i}"
            last = i == c.num_layers - 1
            blk = dict(
                b_qkv=Bv(p + ".attn.to_q", p + ".attn.to_k", p + ".attn.to_v"),
                w_cqkv=W(p + ".attn.add_q_proj", p + ".attn.add_k_proj", p + ".attn.add_v_proj"),
                b_cqkv=Bv(p + ".attn.add_q_proj", p + ".attn.add_k_proj", p + ".attn.add_v_proj"),
                nq=V(p + ".attn.norm_q.weight"), nk=V(p + ".attn.norm_k.weight"),
                cnq=V(p + ".attn.norm_add_q.weight"), cnk=V(p + ".attn.norm_add_k.weight"),
                b_o=Bv(p + ".attn.to_out.0"), b_f1=Bv(p + ".ff.net.0.proj"), b_f2=Bv(p + ".ff.net.2"),
            )
            WQ(blk, "w_qkv", p + ".attn.to_q", p + ".attn.to_k", p + ".attn.to_v")
            WQ(blk, "w_o", p + ".attn.to_out.0")
            WQ(blk, "w_f1", p + ".ff.net.0.proj")
            WQ(blk, "w_f2", p + ".ff.net.2")
            if not last:
                blk.update(w_co=W(p + ".attn.to_add_out"), b_co=Bv(p + ".attn.to_add_out"),
                           w_cf1=W(p + ".ff_context.net.0.proj"), b_cf1=Bv(p + ".ff_context.net.0.proj"),
                           w_cf2=W(p + ".ff_context.net.2"), b_cf2=Bv(p + ".ff_context.net.2"))
            for k2, v2 in blk.items():
                reg(f"blk{i}_{k2}", v2)
            self.blocks.append(blk)

    # ---- plan: ids / 1-axis rope / mask schedule, plus the positional table for this (clips, mask) ---------------------
    def _build_plan(self, clip_shapes, mask_cpu: torch.Tensor) -> SeqPlan:
        # RoPE = ONE 64-wide axis over the running frame index, the time id of the plan
        plan = build_seq_plan(clip_shapes, mask_cpu, (64,), 2, self.device)
        oh, ow = plan.clip_thw[-1][1], plan.clip_thw[-1][2]
        m = self.cfg.pos_embed_max_size
        top, left = (m - oh) // 2, (m - ow) // 2
        base = self.pos_table.reshape(1, m, m, -1)[:, top:top + oh, left:left + ow, :]
        pos = []
        for (t, h, w) in plan.clip_thw:
            e = base
            if (h, w) != (oh, ow):
                e = F.interpolate(base.permute(0, 3, 1, 2), size=(h, w), mode="bilinear").permute(0, 2, 3, 1)
            pos.append(e.reshape(1, h * w, -1).repeat(t, 1, 1).reshape(t * h * w, -1))
        plan.pos = torch.cat(pos, 0).to(self.device).contiguous()
        return plan

    def set_parallel_layout(self, layout) -> None:
        """Attach a `sp.ParallelLayout`: the CFG pair is split first, then the joint sequence is cut into `sp` chunks; q/k/v and
        the attention output cross NVLink as remote stores fused into the QKV-GEMM / attention epilogues (csrc/pf_peer.cu), as
        in B200FluxTransformer.  The reference runs this model with sp 2 or 4 (scripts/inference_multigpu.sh:9); 24 heads
        divide by both, so no head padding is needed."""
        super().set_parallel_layout(layout, "peer")

    def _forward_eager(self, clips, timestep_ratio=None, encoder_hidden_states=None, encoder_attention_mask=None,
                       pooled_projections=None):
        st = StepLaunches(self, clips, encoder_attention_mask)
        d, ranges = st.d, st.ranges
        st.condition(timestep_ratio, pooled_projections)
        st.embed(clips, encoder_hidden_states, x_gate=self.ones_gate)
        for i, w in enumerate(self.blocks):
            last = i == len(self.blocks) - 1
            ov = self.mod_off[f"transformer_blocks.{i}.norm1"]
            oc = self.mod_off[f"transformer_blocks.{i}.norm1_context"]
            # text: AdaLayerNormZero (shift, scale, ...) or, in the last block, AdaLayerNormContinuous (scale, shift)
            if last:
                st.ln_rows(0, oc + d, oc)
            else:
                st.ln_rows(0, oc, oc + d)
            st.ln_rows(1, ov, ov + d)
            for j in (0, 1):
                st.qkv_rows(j, w, (w["w_cqkv"], w["w_qkv"])[j], (w["b_cqkv"], w["b_qkv"])[j], (w["cnq"], w["nq"])[j],
                            (w["cnk"], w["nk"])[j])
            st.attention()
            # context_pre_only: the text stream ends at the last block's attention (MB:659-660)
            st.joint_tail(w, (oc, ov), ((0, 0), ranges[1]) if last else ranges, (w.get("w_co"), w["w_o"]),
                          (w.get("b_co"), w["b_o"]), (w.get("w_cf1"), w["w_f1"]), (w.get("b_cf1"), w["b_f1"]),
                          (w.get("w_cf2"), w["w_f2"]), (w.get("b_cf2"), w["b_f2"]))
        return [st.publish(st.unpatchify(st.head(), clips))]
