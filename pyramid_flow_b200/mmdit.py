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
The workspace gains dit.py's `xn8` (e4m3 twin of `cat`, its first B*S*D bytes also holding the LN-modulate output), `sx8`
and `sc8` (row scales).

use_cuda_graph = True captures each (plan, input shapes and dtypes, precision) once and replays it (graphs.GraphedStep).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import _lib, ops
from ._lib import PF_EPI_GATE_RESID, PF_EPI_GELU_BF16, PF_EPI_QKV_ROPE, PF_EPI_STORE_F32
from .dit import SeqPlan, build_rope_table, check_gemm_precision, fp8_weight, _Cfg
from .graphs import GraphedStep
from dataclasses import dataclass


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


class B200MMDiT(GraphedStep, torch.nn.Module):
    def __init__(self, config: MMDiTConfigB200, state_dict: Dict[str, torch.Tensor], device="cuda",
                 gemm_precision: str = "bf16"):
        super().__init__()
        check_gemm_precision(gemm_precision)
        # "fp8": the block GEMMs listed in the module docstring run on e4m3 operands (opt-in: different numerics)
        self.gemm_precision = gemm_precision
        self.cfg = config
        self.config = _Cfg(in_channels=config.in_channels, num_layers=config.num_layers,
                           num_attention_heads=config.num_attention_heads, attention_head_dim=config.attention_head_dim,
                           joint_attention_dim=config.joint_attention_dim,
                           pooled_projection_dim=config.pooled_projection_dim, patch_size=config.patch_size)
        assert config.attention_head_dim == 64 and config.patch_size == 2
        self._plans, self._ws, self._last_key = {}, {}, None
        self.last_plan: Optional[SeqPlan] = None
        self._import_state_dict(state_dict, torch.device(device))
        self._init_graphs()

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

    @property
    def device(self):
        return self.w_x.device

    @property
    def dtype(self):
        return torch.bfloat16

    def parameters(self, recurse: bool = True):
        return iter([self.w_x])

    # ---- plan: ids / rope / mask schedule / positional table for this (clips, mask) ----------------------------------
    def plan_for(self, clip_shapes, mask: torch.Tensor):
        # fast path keyed on the mask tensor OBJECT (kept alive: its address cannot be recycled), see dit.py
        shapes = tuple(tuple(int(x) for x in s) for s in clip_shapes)
        lk = self._last_key
        if lk is not None and lk[0] is mask and lk[1] == mask._version and lk[2] == shapes:
            return lk[3]
        mask_cpu = mask.detach().to("cpu", torch.int64)
        key = (shapes, mask_cpu.shape, bytes(mask_cpu.numpy().tobytes()))
        hit = self._plans.get(key)
        if hit is None:
            if len(self._plans) >= 16:
                self._plans.clear()
            c = self.cfg
            b, t_len = mask_cpu.shape
            thw = tuple((int(s[-3]), int(s[-2]) // 2, int(s[-1]) // 2) for s in clip_shapes)
            tid = [torch.zeros(t_len)]
            t0 = 0
            pos = []
            oh, ow = thw[-1][1], thw[-1][2]
            m = c.pos_embed_max_size
            top, left = (m - oh) // 2, (m - ow) // 2
            base = self.pos_table.reshape(1, m, m, -1)[:, top:top + oh, left:left + ow, :]
            for (t, h, w) in thw:
                tid.append(torch.arange(t0, t0 + t, dtype=torch.float32)[:, None].repeat(1, h * w).reshape(-1))
                t0 += t
                e = base
                if (h, w) != (oh, ow):
                    e = F.interpolate(base.permute(0, 3, 1, 2), size=(h, w), mode="bilinear").permute(0, 2, 3, 1)
                pos.append(e.reshape(1, h * w, -1).repeat(t, 1, 1).reshape(t * h * w, -1))
            tid = torch.cat(tid)
            video_len = sum(t * h * w for t, h, w in thw)
            seq = t_len + video_len
            seg = torch.arange(1, b + 1, dtype=torch.int32)[:, None].repeat(1, seq)
            seg[:, :t_len][mask_cpu == 0] = 0
            time = tid.to(torch.int32)[None].repeat(b, 1).contiguous()
            sched, pairs = ops.attn_build_schedule(seg, time)
            dev = self.device
            t, h, w = thw[-1]
            plan = SeqPlan(t_len, video_len, seq, t * h * w, thw, build_rope_table(tid[:, None], (64,)).to(dev), seg.to(dev),
                           time.to(dev), sched.to(dev), ops.attn_build_pair_schedule(sched, seq, seg, time).to(dev), int(pairs.sum()))
            hit = (plan, torch.cat(pos, 0).to(dev).contiguous())
            self._plans[key] = hit
        self._last_key = (mask, mask._version, shapes, hit)
        return hit

    def _workspace(self, b: int, plan: SeqPlan, sl: Optional[int] = None) -> dict:
        sl = plan.seq if sl is None else sl
        key = (b, plan.seq, plan.video_len, plan.last_tokens, sl)
        ws = self._ws.get(key)
        if ws is None:
            if len(self._ws) >= 4:
                self._ws.clear()
            c = self.cfg
            d, hn, dev = c.inner_dim, c.num_attention_heads, self.device
            ws = dict(h=torch.empty(b, sl, d, device=dev, dtype=torch.float32),
                      xn=torch.empty(b, sl, d, device=dev, dtype=torch.bfloat16),
                      q=torch.empty(b, hn, sl, 64, device=dev, dtype=torch.bfloat16),
                      k=torch.empty(b, hn, sl, 64, device=dev, dtype=torch.bfloat16),
                      v=torch.empty(b, hn, sl, 64, device=dev, dtype=torch.bfloat16),
                      cat=torch.empty(b, sl, 5 * d, device=dev, dtype=torch.bfloat16),
                      tok=torch.empty(b, plan.video_len, 4 * c.in_channels, device=dev, dtype=torch.bfloat16),
                      mod=torch.empty(b, self.n_mod, device=dev, dtype=torch.float32),
                      temb=torch.empty(b, d, device=dev, dtype=torch.float32),
                      tmp=torch.empty(b, d, device=dev, dtype=torch.float32),
                      head=torch.empty(b, plan.last_tokens, 4 * c.in_channels, device=dev, dtype=torch.float32))
            if self.gemm_precision == "fp8":
                ws["xn8"] = torch.empty(b, sl, 5 * d, device=dev, dtype=torch.float8_e4m3fn)
                ws["sx8"] = torch.empty(b, sl, device=dev, dtype=torch.float32)
                ws["sc8"] = torch.empty(b, sl, device=dev, dtype=torch.float32)
            self._ws[key] = ws
        return ws

    # -- parallel layout (CFG x sequence parallel over NVLink peer memory, sp.py) -----------------------------------------
    def set_parallel_layout(self, layout) -> None:
        """Attach a `sp.ParallelLayout`: the CFG pair is split first, then the joint sequence is cut into `sp` chunks; q/k/v and
        the attention output cross NVLink as remote stores fused into the QKV-GEMM / attention epilogues (csrc/pf_peer.cu), as
        in B200FluxTransformer.  The reference runs this model with sp 2 or 4 (scripts/inference_multigpu.sh:9); 24 heads
        divide by both, so no head padding is needed."""
        if self.gemm_precision == "fp8":
            raise NotImplementedError("gemm_precision='fp8' runs on one GPU only: the sequence-parallel peer-store epilogues "
                                      "have no fp8 form (build the model with gemm_precision='bf16' for a parallel layout)")
        assert self.cfg.num_attention_heads % max(1, layout.sp) == 0, "heads must divide by the SP degree"
        if layout.sp > 1:   # see _lib.load(): one attention kernel for the whole process once sequence parallelism is in play
            _lib.set_option(_lib.PF_OPT_ATTN_TRIPLE_KERNEL, 0)
        self.layout = layout
        self._px = None
        self._graphs.clear()
        self._ws.clear()

    def _peer_exchange(self, plan: SeqPlan):
        """The peer arena (sp.PeerExchange) for this call's shapes; see sp.ensure_peer_exchange."""
        from . import sp as SP
        c = self.cfg
        ct, chh, cww = plan.clip_thw[-1]
        return SP.ensure_peer_exchange(self, self.layout, plan.seq, plan.last_tokens, c.num_attention_heads, 5 * c.inner_dim,
                                       4 * c.in_channels, c.in_channels * ct * chh * 2 * cww * 2 * 4)

    @torch.no_grad()
    def forward(self, sample, timestep_ratio=None, encoder_hidden_states=None, encoder_attention_mask=None,
                pooled_projections=None):
        _lib.require_device()
        assert len(sample) == 1
        clips = sample[0] if isinstance(sample[0], (list, tuple)) else [sample[0]]
        if self.use_cuda_graph:
            return self._forward_graphed(list(clips), timestep_ratio, encoder_hidden_states, encoder_attention_mask,
                                         pooled_projections)
        return self._forward_eager(clips, timestep_ratio, encoder_hidden_states, encoder_attention_mask, pooled_projections)

    # -- CUDA-graph replay (graphs.GraphedStep) -------------------------------------------------------------------------
    def _graph_plan(self, clips, mask):   # (plan, positional table): the captured device copy into `h` reads the table
        return self.plan_for([cl.shape for cl in clips], mask)

    def _graph_key_fields(self) -> tuple:
        return (self.gemm_precision,)

    def _graph_prealloc(self, plan: SeqPlan, clips) -> None:
        lay = getattr(self, "layout", None)
        if lay is not None and lay.enabled:
            from . import sp as SP
            c0, c1 = SP.chunk_bounds(plan.seq, lay.sp, lay.sp_rank)
            self._workspace(1, plan, c1 - c0)
            self._peer_exchange(plan)
        else:
            self._workspace(clips[-1].shape[0], plan)

    def _forward_eager(self, clips, timestep_ratio=None, encoder_hidden_states=None, encoder_attention_mask=None,
                       pooled_projections=None):
        c = self.cfg
        d, hn = c.inner_dim, c.num_attention_heads
        bg = clips[-1].shape[0]
        plan, pos = self.plan_for([cl.shape for cl in clips], encoder_attention_mask)
        self.last_plan = plan
        t_len, s, lv = plan.text_len, plan.seq, plan.video_len
        lay = getattr(self, "layout", None)
        par = lay is not None and lay.enabled
        if par:
            from . import sp as SP
            assert bg == lay.cfg_ways, "CFG-parallel layout expects the [uncond ; cond] batch"
            b, b0, nsp = 1, lay.cfg_rank, lay.sp
            c0, c1 = SP.chunk_bounds(s, nsp, lay.sp_rank)
        else:
            b, b0, nsp, c0, c1 = bg, 0, 1, 0, s
        sl = c1 - c0
        ws = self._workspace(b, plan, sl)
        h, xn, q, k, v, cat, mod = ws["h"], ws["xn"], ws["q"], ws["k"], ws["v"], ws["cat"], ws["mod"]
        nm = self.n_mod
        ldc = 5 * d
        px = None
        if par:
            px = self._peer_exchange(plan)
            if nsp > 1:
                cat = px.cat(sl)
                qkv_x = px.qkv(s)
        rope = plan.rope[c0:c1]
        tb, te = max(0, c0), min(t_len, c1)
        vb, ve = max(t_len, c0), min(s, c1)
        ranges = ((tb - c0, max(0, te - tb)), (vb - c0, max(0, ve - vb)))        # (text, video) rows of my chunk

        t32 = timestep_ratio.detach().to(device=self.device, dtype=torch.float32)[b0:b0 + b].contiguous()
        tproj = ops.timestep_embedding(t32, 256, round_bf16=False)
        ops.small_linear(tproj, self.w_t1, self.b_t1, ws["tmp"], act_out=1)
        ops.small_linear(ws["tmp"], self.w_t2, self.b_t2, ws["temb"])
        pooled = pooled_projections.detach().to(device=self.device, dtype=torch.float32)[b0:b0 + b].contiguous()
        ops.small_linear(pooled, self.w_p1, self.b_p1, ws["tmp"], act_out=1)
        ops.small_linear(ws["tmp"], self.w_p2, self.b_p2, ws["temb"], accumulate=True)
        ops.small_linear(ws["temb"], self.w_mod, self.b_mod, mod, act_in=1)

        if ranges[0][1] > 0:
            enc = encoder_hidden_states.detach().to(device=self.device, dtype=torch.bfloat16)[b0:b0 + b].contiguous()
            ops.gemm(enc, self.w_ctx, self.b_ctx, PF_EPI_STORE_F32, batches=b, rows_per_batch=t_len, row_begin=tb,
                     row_count=te - tb, out=h, ldo=d, out_batch_rows=sl, out_row_begin=tb - c0)
        if ranges[1][1] > 0:
            tok0 = 0
            for cl, (ct, chh, cww) in zip(clips, plan.clip_thw):
                cl = cl.detach()[b0:b0 + b]
                if cl.dtype not in (torch.float32, torch.bfloat16):
                    cl = cl.float()
                ops.patchify(cl.contiguous(), ws["tok"], lv, tok0)
                tok0 += ct * chh * cww
            # the sincos table is placed in the stream first (device copy), the patch-embed GEMM accumulates onto it
            h[:, vb - c0:ve - c0].copy_(pos[None, vb - t_len:ve - t_len].expand(b, -1, -1))
            ops.gemm(ws["tok"], self.w_x, self.b_x, PF_EPI_GATE_RESID, batches=b, rows_per_batch=lv, row_begin=vb - t_len,
                     row_count=ve - vb, out=h, ldo=d, out_batch_rows=sl, out_row_begin=vb - c0, gate=self.ones_gate,
                     gate_batch_stride=0)

        def lnmod(off_shift, off_scale, r0, rc):
            if rc > 0:
                ops.ln_modulate(h, xn, mod[:, off_shift:], mod[:, off_scale:], nm, batches=b, rows_per_batch=sl, row_begin=r0,
                                row_count=rc)

        fp8 = self.gemm_precision == "fp8"       # single GPU only (set_parallel_layout), so the video rows are ranges[1]
        if fp8:
            xn8, sx8, sc8 = ws["xn8"], ws["sx8"], ws["sc8"]
            xa8 = xn8.view(-1)[:b * sl * d].view(b, sl, d)    # LN-modulate output, row stride d (module docstring)

        def lnmod8(off_shift, off_scale, r0, rc):
            ops.ln_modulate_fp8(h, xa8, sx8, mod[:, off_shift:], mod[:, off_scale:], nm, batches=b, rows_per_batch=sl,
                                row_begin=r0, row_count=rc)

        def quant8(col0, col1, r0, rc):   # cat[:, r0:r0 + rc, col0:col1] -> the same block of xn8, row scales -> sc8
            ops.quantize_rows_fp8(cat[:, :, col0:col1], xn8[:, :, col0:col1], sc8, batches=b, rows_per_batch=sl, row_begin=r0,
                                  row_count=rc)

        peer_qkv = None
        if px is not None and nsp > 1:
            peer_qkv = dict(peer_ptrs=[pp + px.off_qkv for pp in px.sp_buf.ptrs], peer_heads=hn // nsp, peer_seq=s, peer_row0=c0)
        seg, tim, sched, sched2 = plan.seg[b0:b0 + b], plan.time[b0:b0 + b], plan.sched[b0:b0 + b], plan.sched2[b0:b0 + b]
        scale = 1.0 / math.sqrt(64)
        for i, w in enumerate(self.blocks):
            last = i == c.num_layers - 1
            ov = self.mod_off[f"transformer_blocks.{i}.norm1"]
            oc = self.mod_off[f"transformer_blocks.{i}.norm1_context"]
            offs = (oc, ov)
            # text: AdaLayerNormZero (shift, scale, ...) or, in the last block, AdaLayerNormContinuous (scale, shift)
            if last:
                lnmod(oc + d, oc, *ranges[0])
            else:
                lnmod(oc, oc + d, *ranges[0])
            if fp8 and ranges[1][1] > 0:
                lnmod8(ov, ov + d, *ranges[1])
            else:
                lnmod(ov, ov + d, *ranges[1])
            for j, (r0, rc) in enumerate(ranges):
                if fp8 and j == 1 and rc > 0:
                    ops.gemm_fp8(xa8, sx8, w["w_qkv"], w["s_qkv"], w["b_qkv"], PF_EPI_QKV_ROPE, batches=b, rows_per_batch=sl,
                                 row_begin=r0, row_count=rc, q_out=q, k_out=k, v_out=v, rope=rope, q_norm_w=w["nq"],
                                 k_norm_w=w["nk"], norm_eps=1e-5, heads=hn, head_dim=64, seq_len=sl)
                elif rc > 0:
                    ops.gemm(xn, (w["w_cqkv"], w["w_qkv"])[j], (w["b_cqkv"], w["b_qkv"])[j], PF_EPI_QKV_ROPE, batches=b,
                             rows_per_batch=sl, row_begin=r0, row_count=rc, q_out=q, k_out=k, v_out=v, rope=rope,
                             q_norm_w=(w["cnq"], w["nq"])[j], k_norm_w=(w["cnk"], w["nk"])[j], norm_eps=1e-5, heads=hn,
                             head_dim=64, seq_len=sl, peer=peer_qkv)
            if nsp == 1:
                ops.attn_fwd(q, k, v, cat, seg, tim, sched, scale, pair_sched=sched2)
            else:
                px.barrier_sp()                    # every rank's QKV epilogue has stored into every rank's gathered buffer
                ops.attn_fwd(qkv_x[0][None], qkv_x[1][None], qkv_x[2][None], None, seg, tim, sched, scale, pair_sched=sched2,
                             ldo=ldc, peer=dict(peer_ptrs=[pp + px.off_cat for pp in px.sp_buf.ptrs], peer_chunk_rows=sl,
                                                peer_col_begin=lay.sp_rank * (hn // nsp) * 64))
                px.barrier_sp()                    # ... and every rank's attention epilogue into every rank's `cat`
            for j, (r0, rc) in enumerate(ranges):
                if rc == 0 or (j == 0 and last):
                    continue   # context_pre_only: the text stream ends here (MB:659-660)
                if fp8 and j == 1:
                    rows = dict(batches=b, rows_per_batch=sl, row_begin=r0, row_count=rc)
                    quant8(0, d, r0, rc)
                    ops.gemm_fp8(xn8[:, :, :d], sc8, w["w_o"], w["s_o"], w["b_o"], PF_EPI_GATE_RESID, out=h, ldo=d,
                                 gate=mod[:, offs[j] + 2 * d:], gate_batch_stride=nm, **rows)
                    lnmod8(offs[j] + 3 * d, offs[j] + 4 * d, r0, rc)
                    ops.gemm_fp8(xa8, sx8, w["w_f1"], w["s_f1"], w["b_f1"], PF_EPI_GELU_BF16, out=cat, ldo=ldc, out_col_begin=d,
                                 **rows)
                    quant8(d, ldc, r0, rc)
                    ops.gemm_fp8(xn8[:, :, d:], sc8, w["w_f2"], w["s_f2"], w["b_f2"], PF_EPI_GATE_RESID, out=h, ldo=d,
                                 gate=mod[:, offs[j] + 5 * d:], gate_batch_stride=nm, **rows)
                    continue
                wo, bo = ((w.get("w_co"), w["w_o"])[j], (w.get("b_co"), w["b_o"])[j])
                wf1, bf1 = ((w.get("w_cf1"), w["w_f1"])[j], (w.get("b_cf1"), w["b_f1"])[j])
                wf2, bf2 = ((w.get("w_cf2"), w["w_f2"])[j], (w.get("b_cf2"), w["b_f2"])[j])
                ops.gemm(cat[:, :, :d], wo, bo, PF_EPI_GATE_RESID, batches=b, rows_per_batch=sl, row_begin=r0, row_count=rc,
                         out=h, ldo=d, gate=mod[:, offs[j] + 2 * d:], gate_batch_stride=nm)
                lnmod(offs[j] + 3 * d, offs[j] + 4 * d, r0, rc)
                ops.gemm(xn, wf1, bf1, PF_EPI_GELU_BF16, batches=b, rows_per_batch=sl, row_begin=r0, row_count=rc, out=cat,
                         ldo=ldc, out_col_begin=d)
                ops.gemm(cat[:, :, d:], wf2, bf2, PF_EPI_GATE_RESID, batches=b, rows_per_batch=sl, row_begin=r0, row_count=rc,
                         out=h, ldo=d, gate=mod[:, offs[j] + 5 * d:], gate_batch_stride=nm)

        n_last = plan.last_tokens
        o = self.mod_off["norm_out"]
        g0, g1 = max(s - n_last, c0), c1                 # my part of the last n_last tokens
        head = ws["head"]
        peer_head = px is not None and nsp > 1
        if peer_head:
            head = px.head(n_last)
        if g1 > g0:
            lnmod(o + d, o, g0 - c0, g1 - g0)
            ops.gemm(xn, self.w_out, self.b_out, PF_EPI_STORE_F32, batches=b, rows_per_batch=sl, row_begin=g0 - c0,
                     row_count=g1 - g0, out=head, ldo=4 * c.in_channels, out_batch_rows=n_last, out_row_begin=g0 - (s - n_last))
            if peer_head:
                r0h = g0 - (s - n_last)
                px.bcast(px.sp_buf, head[0, r0h:r0h + (g1 - g0)], px.off_head + r0h * 4 * c.in_channels * 4)
        if peer_head:
            px.barrier_sp()
        ct, chh, cww = plan.clip_thw[-1]
        odt = clips[-1].dtype if clips[-1].dtype in (torch.float32, torch.bfloat16) else torch.float32
        out = torch.empty(b, c.in_channels, ct, chh * 2, cww * 2, device=self.device, dtype=odt)
        ops.unpatchify(head, n_last, 0, out)
        if par:
            vel = px.vel((bg, *out.shape[1:]), odt)
            if lay.sp_rank == 0:
                px.bcast(px.world_buf, out.view(-1), px.w_off_vel + lay.cfg_rank * px.vel_bytes)
            px.barrier_world()
            out = vel.clone()
        return [out]
