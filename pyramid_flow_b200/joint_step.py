"""The step scaffolding shared by the two joint-attention DiT drop-ins, `dit.B200FluxTransformer` (miniFLUX) and
`mmdit.B200MMDiT` (SD3): the plan cache, the workspace, the CFG x sequence-parallel layout, the eager / CUDA-graph dispatch,
and, in `StepLaunches`, the launches of one step that both models make in the same form.

A model supplies its weights and the data in which the two differ: `token_dim` (features of one patch token: the patchify
output and the head's output width), `norm_eps` (q/k RMSNorm of the QKV epilogue), `_build_plan` (ids, RoPE table and, for
the SD3 model, the positional table the patch embed accumulates onto), and its own `_forward_eager`, which walks its blocks
with the `StepLaunches` helpers.

Data layout in HBM (B = CFG batch, S = text + all clip tokens, D = heads*64, Hp = heads, padded under sequence parallelism):
  h    fp32 [B, S, D]      joint residual stream ([text ; clip_0 ; ... ; clip_n] per sample) — fp32 so that the residual
                           adds of every block do not accumulate bf16 rounding (the reference keeps it bf16)
  xn   bf16 [B, S, D]      LN+modulated activations (GEMM A operand)
  q,k,v bf16 [B, Hp, S, 64] head-major, written by the QKV epilogue, read by TMA in the attention kernel
  cat  bf16 [B, S, Hp*64 + 4D]  [attention out | MLP hidden]: FF2 (and miniFLUX's single-block proj_out) read it in place
  mod  fp32 [B, N_mod]     every layer's (shift, scale, gate, ...) from ONE GEMV per step
  fp8 only:
  xn8  e4m3 [B, S, 5D]     twin of `cat`: quantised [attention out | MLP hidden] rows; its first B*S*D bytes also hold the
                           LN-modulate output [B, S, D] (consumed by QKV / FF1 / proj_mlp before the twin is refilled)
  sx8, sc8 fp32 [B, S]     row scales of the LN-modulate output and of the quantised `cat` rows
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import torch

from . import _lib, ops
from ._lib import PF_EPI_GATE_RESID, PF_EPI_GELU_BF16, PF_EPI_QKV_ROPE, PF_EPI_STORE_F32
from .graphs import GraphedStep

# default formulation of the sequence-parallel exchange: "peer" (remote stores fused into the kernels over NVLink peer memory)
# or "nccl" (all_to_all_single, miniFLUX only)
DEFAULT_EXCHANGE = "peer"
_ATTN_SCALE = 1.0 / math.sqrt(64)    # head_dim 64


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def fp8_weight(sd: Dict[str, torch.Tensor], names: Sequence[str], device):
    """The state-dict weights `names` concatenated along the output dim, quantised once on the host from their fp32 values:
    (e4m3 [N, K], fp32 per-output-channel scale [N]) on `device`; no bf16 copy is kept."""
    w8, sc = ops.quantize_weight_fp8(torch.cat([sd[n + ".weight"].float().cpu() for n in names], 0))
    return w8.to(device), sc.to(device)


class _KernelTimer:
    """Optional CUDA-event timing of kernel families inside a step (bench.py breakdown); disabled => zero overhead."""

    def __init__(self):
        self.enabled = False
        self.events = []

    def __call__(self, tag: str):
        return _Span(self, tag) if self.enabled else _NULL_SPAN

    def totals_ms(self):
        out = {}
        for tag, e0, e1 in self.events:
            out[tag] = out.get(tag, 0.0) + e0.elapsed_time(e1)
        return out


class _Span:
    def __init__(self, timer, tag):
        self.t, self.tag = timer, tag

    def __enter__(self):
        self.e0 = torch.cuda.Event(enable_timing=True)
        self.e0.record()

    def __exit__(self, *a):
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        self.t.events.append((self.tag, self.e0, e1))


class _NullSpan:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


_NULL_SPAN = _NullSpan()


class JointStep(GraphedStep, torch.nn.Module):
    """Base of the two DiT drop-ins: packed weights are imported by the model, the step is a fixed kernel-launch sequence."""

    norm_eps = 1e-6       # q/k RMSNorm eps of the QKV epilogue

    def __init__(self, config, gemm_precision: str):
        super().__init__()
        if gemm_precision not in ("bf16", "fp8"):
            raise ValueError(f"gemm_precision must be 'bf16' or 'fp8', not {gemm_precision!r}")
        # "fp8": the block GEMMs listed in the model's docstring run on e4m3 operands (opt-in: different numerics)
        self.gemm_precision = gemm_precision
        self.cfg = config
        assert config.attention_head_dim == 64, "kernels are specialised for head_dim 64"
        self._plans: Dict[tuple, object] = {}
        self._ws: Dict[tuple, dict] = {}
        self._last_key = None
        self.last_plan = None
        self.emulate_bf16_rounding = False   # miniFLUX: the reference's bf16 rounding of the sinusoidal projection
        self.output_fp32 = False        # fused CFG+Euler path of the sampler keeps the velocity in fp32
        self.attn_events = None         # bench.py: list collecting (start, end) CUDA events around every attention launch
        self.timer = _KernelTimer()
        self.attn_variant = 0           # pf_attn_desc.variant (every value runs the one sm_90a kernel)
        self.layout, self.exchange, self._px = None, DEFAULT_EXCHANGE, None
        self._hp = config.num_attention_heads
        self._init_graphs()             # use_cuda_graph: the launches of a step captured once per shape (graphs.py)

    @property
    def device(self):
        return self.w_x.device

    @property
    def dtype(self):
        return torch.bfloat16

    def parameters(self, recurse: bool = True):  # the pipeline only asks next(self.dit.parameters()).device/.dtype
        return iter([self.w_x])

    # -- plan ----------------------------------------------------------------------------------------------------------
    def plan_for(self, clip_shapes, mask: torch.Tensor):
        """The model's SeqPlan for these clip shapes and text mask (built by `_build_plan`, cached)."""
        # fast path: the SAME mask tensor object (kept alive here, so its address cannot be recycled by the caching
        # allocator for a different mask), unmodified since, and the same clip shapes as the previous call -> no D2H sync
        shapes = tuple(tuple(int(x) for x in s) for s in clip_shapes)
        lk = self._last_key
        if lk is not None and lk[0] is mask and lk[1] == mask._version and lk[2] == shapes:
            return lk[3]
        mask_cpu = mask.detach().to("cpu", torch.int64)
        key = (shapes, mask_cpu.shape, bytes(mask_cpu.numpy().tobytes()))
        plan = self._plans.get(key)
        if plan is None:
            if len(self._plans) >= 16:
                self._plans.clear()
            plan = self._build_plan(clip_shapes, mask_cpu)
            self._plans[key] = plan
        self._last_key = (mask, mask._version, shapes, plan)
        return plan

    # -- workspace -----------------------------------------------------------------------------------------------------
    def _workspace(self, b: int, plan, sl: Optional[int] = None, hp: Optional[int] = None) -> dict:
        c = self.cfg
        sl = plan.seq if sl is None else sl
        hp = c.num_attention_heads if hp is None else hp
        key = (b, plan.seq, plan.video_len, plan.last_tokens, sl, hp)
        ws = self._ws.get(key)
        if ws is None:
            if len(self._ws) >= 4:   # shapes change every unit/stage; keep the cache bounded
                self._ws.clear()
            d, hn, tw, dev = c.inner_dim, c.num_attention_heads, self.token_dim, self.device
            alloc = torch.zeros if hp != hn else torch.empty      # padded heads must read as zeros
            ws = dict(
                h=torch.empty(b, sl, d, device=dev, dtype=torch.float32),
                xn=torch.empty(b, sl, d, device=dev, dtype=torch.bfloat16),
                q=alloc(b, hp, sl, 64, device=dev, dtype=torch.bfloat16),
                k=alloc(b, hp, sl, 64, device=dev, dtype=torch.bfloat16),
                v=alloc(b, hp, sl, 64, device=dev, dtype=torch.bfloat16),
                cat=torch.empty(b, sl, hp * 64 + 4 * d, device=dev, dtype=torch.bfloat16),
                tok=torch.empty(b, plan.video_len, tw, device=dev, dtype=torch.bfloat16),
                mod=torch.empty(b, self.n_mod, device=dev, dtype=torch.float32),
                temb=torch.empty(b, d, device=dev, dtype=torch.float32),
                tmp=torch.empty(b, d, device=dev, dtype=torch.float32),
                head=torch.zeros(b, plan.last_tokens, tw, device=dev, dtype=torch.float32),
            )
            if self.gemm_precision == "fp8":
                ws["xn8"] = torch.empty(b, sl, hp * 64 + 4 * d, device=dev, dtype=torch.float8_e4m3fn)
                ws["sx8"] = torch.empty(b, sl, device=dev, dtype=torch.float32)
                ws["sc8"] = torch.empty(b, sl, device=dev, dtype=torch.float32)
            self._ws[key] = ws
        return ws

    # -- parallel layout (CFG x sequence parallel, sp.py) ---------------------------------------------------------------
    def set_parallel_layout(self, layout, exchange: str = DEFAULT_EXCHANGE) -> None:
        """Attach a `sp.ParallelLayout` (after torch.distributed is initialised); weights are replicated.
        exchange = "peer": q/k/v and the attention output cross NVLink as remote stores fused into the QKV GEMM / attention
        epilogues + flag barriers (csrc/pf_peer.cu): no NCCL call in the step, CUDA-graph capturable.  "nccl": the
        all_to_all_single formulation (miniFLUX, kept for A/B measurements)."""
        if self.gemm_precision == "fp8":
            raise NotImplementedError("gemm_precision='fp8' runs on one GPU only: the sequence-parallel peer-store epilogues "
                                      "have no fp8 form (build the model with gemm_precision='bf16' for a parallel layout)")
        assert exchange in ("peer", "nccl")
        from .sp import padded_heads
        hp = padded_heads(self.cfg.num_attention_heads, layout.sp)
        if hp != self.cfg.num_attention_heads:
            self._pad_heads(hp)
        if layout.sp > 1:   # see _lib.load(): one attention kernel for the whole process once sequence parallelism is in play
            _lib.set_option(_lib.PF_OPT_ATTN_TRIPLE_KERNEL, 0)
        self.layout, self.exchange, self._px, self._hp = layout, exchange, None, hp
        self._graphs.clear()
        self._ws.clear()

    def _pad_heads(self, hp: int) -> None:
        raise AssertionError("heads must divide by the SP degree")

    def _peer_exchange(self, plan):
        """The peer arena (sp.PeerExchange) for this call's shapes; see sp.ensure_peer_exchange."""
        from . import sp as SP
        hp, tw = self._hp, self.token_dim
        ct, chh, cww = plan.clip_thw[-1]
        return SP.ensure_peer_exchange(self, self.layout, plan.seq, plan.last_tokens, hp, hp * 64 + 4 * self.cfg.inner_dim,
                                       tw, (tw // 4) * ct * chh * 2 * cww * 2 * 4)

    # -- the step ------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, sample, timestep_ratio=None, encoder_hidden_states=None, encoder_attention_mask=None,
                pooled_projections=None):
        _lib.require_device()
        assert len(sample) == 1, "inference passes one stage per call (pipeline P:760-766)"
        clips = sample[0] if isinstance(sample[0], (list, tuple)) else [sample[0]]
        lay = self.layout
        # the NCCL formulation of the parallel step stays host-launched (its all-to-alls are not captured); the peer-memory
        # formulation is plain kernels and is captured like the single-GPU step
        nccl_par = lay is not None and lay.enabled and self.exchange == "nccl"
        if self.use_cuda_graph and not nccl_par and not self.timer.enabled and self.attn_events is None:
            return self._forward_graphed(list(clips), timestep_ratio, encoder_hidden_states, encoder_attention_mask,
                                         pooled_projections)
        return self._forward_eager(clips, timestep_ratio, encoder_hidden_states, encoder_attention_mask,
                                   pooled_projections)

    # -- CUDA-graph replay (graphs.GraphedStep) -------------------------------------------------------------------------
    def _graph_key_fields(self) -> tuple:
        return (self.gemm_precision, bool(self.output_fp32), bool(self.emulate_bf16_rounding), int(self.attn_variant))

    def _graph_prealloc(self, plan, clips) -> None:
        lay = self.layout
        if lay is not None and lay.enabled:
            from . import sp as SP
            c0, c1 = SP.chunk_bounds(plan.seq, lay.sp, lay.sp_rank)
            self._workspace(1, plan, c1 - c0, self._hp)
            if self.exchange == "peer":
                self._peer_exchange(plan)
        else:
            self._workspace(clips[-1].shape[0], plan)


def row_ranges(text_len: int, seq: int, c0: int, c1: int):
    """Local (row_begin, row_count) of the (text, video) parts of the token chunk [c0, c1) of the joint sequence."""
    tb, te = max(0, c0), min(text_len, c1)
    vb, ve = max(text_len, c0), min(seq, c1)
    return ((tb - c0, max(0, te - tb)), (vb - c0, max(0, ve - vb)))


class StepLaunches:
    """One call's rows, buffers and exchange arena, and the launches both models make in the same form.

    Rows: the CFG batch `bg`; this rank's `b` samples from `b0`; its token chunk [c0, c1) of the joint sequence (`sl` rows);
    `ranges` = local (row_begin, row_count) of the (text, video) parts of the chunk.  With a parallel layout every rank runs
    one CFG branch on one chunk; with the peer exchange `cat` and the gathered q/k/v live in the peer arena."""

    def __init__(self, m: JointStep, clips, mask):
        c = m.cfg
        self.m, self.T, self.d, self.hn, self.nm = m, m.timer, c.inner_dim, c.num_attention_heads, m.n_mod
        self.lay = lay = m.layout
        self.par = par = lay is not None and lay.enabled
        self.bg = clips[-1].shape[0]                        # global (CFG) batch
        self.plan = plan = m.plan_for([cl.shape for cl in clips], mask)
        m.last_plan = plan
        t_len, s = plan.text_len, plan.seq
        if par:
            from . import sp as SP
            assert self.bg == lay.cfg_ways, "CFG-parallel layout expects the [uncond ; cond] batch"
            b, b0, nsp, hp = 1, lay.cfg_rank, lay.sp, m._hp          # this rank's CFG branch
            c0, c1 = SP.chunk_bounds(s, nsp, lay.sp_rank)
        else:
            b, b0, nsp, hp, c0, c1 = self.bg, 0, 1, self.hn, 0, s
        self.b, self.b0, self.nsp, self.hp, self.c0, self.c1 = b, b0, nsp, hp, c0, c1
        self.sl = sl = c1 - c0                               # tokens of the joint sequence owned by this rank
        self.wa = wa = hp * 64                               # width of the attention block in `cat`
        self.ldc = ldc = wa + 4 * self.d
        self.ws = ws = m._workspace(b, plan, sl, hp)
        self.h, self.xn, self.q, self.k, self.v, self.cat, self.mod = (ws["h"], ws["xn"], ws["q"], ws["k"], ws["v"],
                                                                       ws["cat"], ws["mod"])
        self.px = px = m._peer_exchange(plan) if (par and m.exchange == "peer") else None
        self.peer_qkv = self.peer_out = None
        if px is not None and nsp > 1:
            self.cat = px.cat(sl)
            self.qkv_x = px.qkv(s)                           # [3, Hg, S, 64]: my head group over the whole sequence
            self.peer_qkv, self.peer_out = SP.peer_store_args(s, nsp, lay.sp_rank, hp,
                                                              [pp + px.off_qkv for pp in px.sp_buf.ptrs],
                                                              [pp + px.off_cat for pp in px.sp_buf.ptrs])
        self.rope = plan.rope[c0:c1]
        self.ranges = row_ranges(t_len, s, c0, c1)
        self.seg, self.tim = plan.seg[b0:b0 + b], plan.time[b0:b0 + b]
        self.sched, self.sched2 = plan.sched[b0:b0 + b], plan.sched2[b0:b0 + b]
        self.fp8 = m.gemm_precision == "fp8"
        if self.fp8:
            self.xn8, self.sx8, self.sc8 = ws["xn8"], ws["sx8"], ws["sc8"]
            self.xa8 = self.xn8.view(-1)[:b * sl * self.d].view(b, sl, self.d)   # LN-modulate output, row stride d

    # ---- conditioning (E:193-201): timestep arrives already rounded to bf16 by the pipeline (P:750)
    def condition(self, timestep_ratio, pooled_projections) -> None:
        m, ws, b0, b = self.m, self.ws, self.b0, self.b
        t32 = timestep_ratio.detach().to(device=m.device, dtype=torch.float32)[b0:b0 + b].contiguous()
        tproj = ops.timestep_embedding(t32, 256, round_bf16=m.emulate_bf16_rounding)
        ops.small_linear(tproj, m.w_t1, m.b_t1, ws["tmp"], act_out=1)
        ops.small_linear(ws["tmp"], m.w_t2, m.b_t2, ws["temb"])
        pooled = pooled_projections.detach().to(device=m.device, dtype=torch.float32)[b0:b0 + b].contiguous()
        ops.small_linear(pooled, m.w_p1, m.b_p1, ws["tmp"], act_out=1)
        ops.small_linear(ws["tmp"], m.w_p2, m.b_p2, ws["temb"], accumulate=True)
        # every AdaLN modulation of the step in one GEMV: mod = Linear(SiLU(temb)) for all layers
        ops.small_linear(ws["temb"], m.w_mod, m.b_mod, self.mod, act_in=1)

    def embed(self, clips, encoder_hidden_states, x_gate: Optional[torch.Tensor] = None) -> None:
        """The embedders write straight into the joint fp32 residual stream (only this rank's rows).  x_gate = None: the
        patch-embed GEMM stores its rows; a ones vector: it accumulates onto the plan's positional table, placed there first."""
        m, plan, b0, b, h, d, sl, c0 = self.m, self.plan, self.b0, self.b, self.h, self.d, self.sl, self.c0
        t_len, lv = plan.text_len, plan.video_len
        (tr, tc), (vr, vc) = self.ranges
        if tc > 0:
            enc = encoder_hidden_states.detach().to(device=m.device, dtype=torch.bfloat16)[b0:b0 + b].contiguous()
            ops.gemm(enc, m.w_ctx, m.b_ctx, PF_EPI_STORE_F32, batches=b, rows_per_batch=t_len, row_begin=tr + c0,
                     row_count=tc, out=h, ldo=d, out_batch_rows=sl, out_row_begin=tr)
        if vc > 0:
            tok0 = 0
            for cl, (ct, chh, cww) in zip(clips, plan.clip_thw):
                cl = cl.detach()[b0:b0 + b]
                if cl.dtype not in (torch.float32, torch.bfloat16):
                    cl = cl.float()
                ops.patchify(cl.contiguous(), self.ws["tok"], lv, tok0)
                tok0 += ct * chh * cww
            vb = vr + c0 - t_len                             # first video token of my chunk
            if x_gate is not None:
                h[:, vr:vr + vc].copy_(plan.pos[None, vb:vb + vc].expand(b, -1, -1))
            ops.gemm(self.ws["tok"], m.w_x, m.b_x, PF_EPI_STORE_F32 if x_gate is None else PF_EPI_GATE_RESID, batches=b,
                     rows_per_batch=lv, row_begin=vb, row_count=vc, out=h, ldo=d, out_batch_rows=sl, out_row_begin=vr,
                     gate=x_gate, gate_batch_stride=0)

    # ---- LN-modulate, QKV, row quantiser: one launch each
    def ln(self, off_shift, off_scale, r0, rc) -> None:
        if rc > 0:
            mod = self.mod
            with self.T("ln_modulate"):
                ops.ln_modulate(self.h, self.xn, mod[:, off_shift:], mod[:, off_scale:], self.nm, batches=self.b,
                                rows_per_batch=self.sl, row_begin=r0, row_count=rc)

    def ln8(self, off_shift, off_scale, r0, rc) -> None:
        mod = self.mod
        with self.T("ln_modulate"):
            ops.ln_modulate_fp8(self.h, self.xa8, self.sx8, mod[:, off_shift:], mod[:, off_scale:], self.nm, batches=self.b,
                                rows_per_batch=self.sl, row_begin=r0, row_count=rc)

    def quant8(self, col0, col1, r0, rc) -> None:   # cat[:, r0:r0 + rc, col0:col1] -> the same block of xn8, row scales -> sc8
        with self.T("quantize_fp8"):
            ops.quantize_rows_fp8(self.cat[:, :, col0:col1], self.xn8[:, :, col0:col1], self.sc8, batches=self.b,
                                  rows_per_batch=self.sl, row_begin=r0, row_count=rc)

    def qkv(self, wq, bq, nq, nk, r0, rc) -> None:
        if rc > 0:
            with self.T("gemm_qkv"):
                ops.gemm(self.xn, wq, bq, PF_EPI_QKV_ROPE, batches=self.b, rows_per_batch=self.sl, row_begin=r0, row_count=rc,
                         q_out=self.q, k_out=self.k, v_out=self.v, rope=self.rope, q_norm_w=nq, k_norm_w=nk,
                         norm_eps=self.m.norm_eps, heads=self.hn, head_dim=64, seq_len=self.sl, peer=self.peer_qkv)

    def qkv8(self, wq, sq, bq, nq, nk, r0, rc) -> None:
        with self.T("gemm_qkv"):
            ops.gemm_fp8(self.xa8, self.sx8, wq, sq, bq, PF_EPI_QKV_ROPE, batches=self.b, rows_per_batch=self.sl,
                         row_begin=r0, row_count=rc, q_out=self.q, k_out=self.k, v_out=self.v, rope=self.rope, q_norm_w=nq,
                         k_norm_w=nk, norm_eps=self.m.norm_eps, heads=self.hn, head_dim=64, seq_len=self.sl)

    # the text (j = 0) or video (j = 1) rows of a joint block; under gemm_precision="fp8" the video rows run on e4m3
    def ln_rows(self, j, off_shift, off_scale) -> None:
        r0, rc = self.ranges[j]
        if self.fp8 and j == 1 and rc > 0:
            self.ln8(off_shift, off_scale, r0, rc)
        else:
            self.ln(off_shift, off_scale, r0, rc)

    def qkv_rows(self, j, w, wq, bq, nq, nk) -> None:
        r0, rc = self.ranges[j]
        if self.fp8 and j == 1 and rc > 0:
            self.qkv8(w["w_qkv"], w["s_qkv"], bq, nq, nk, r0, rc)
        else:
            self.qkv(wq, bq, nq, nk, r0, rc)

    # ---- masked joint attention
    def attn(self, q, k, v, out, q_row_begin=0, ldo=None, peer=None) -> None:
        """One attention launch on this call's plan, bracketed by CUDA events when `attn_events` collects them."""
        ev = self.m.attn_events
        if ev is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        ops.attn_fwd(q, k, v, out, self.seg, self.tim, self.sched, _ATTN_SCALE, variant=self.m.attn_variant,
                     q_row_begin=q_row_begin, pair_sched=self.sched2, ldo=ldo, peer=peer)
        if ev is not None:
            e1.record()
            ev.append((e0, e1))

    def attention(self, q_row_begin=0) -> None:
        """Attention output of this rank's rows into `cat[:, :, :wa]`: on one GPU, or across the sp group in peer memory."""
        if self.nsp == 1:
            self.attn(self.q, self.k, self.v, self.cat, q_row_begin)
            return
        # every rank's QKV epilogue has stored into every rank's gathered buffer: order those stores before the reads; the
        # second barrier orders the attention epilogue's stores into every rank's `cat` before the projections that read it
        qkv_x = self.qkv_x
        self.px.barrier_sp()
        self.attn(qkv_x[0][None], qkv_x[1][None], qkv_x[2][None], None, q_row_begin, ldo=self.ldc, peer=self.peer_out)
        self.px.barrier_sp()

    def joint_tail(self, w, offs, ranges, wo, bo, wf1, bf1, wf2, bf2) -> None:
        """After attention, per (text, video) range of `ranges` with (modulation offset, weights, biases) of that stream:
        attn-out GEMM (+gate*x+residual), LN-modulate, FF1 GEMM (+GELU) into `cat`, FF2 GEMM (+gate, residual)."""
        T, b, sl, h, xn, cat, mod, nm, d, wa, ldc = (self.T, self.b, self.sl, self.h, self.xn, self.cat, self.mod, self.nm,
                                                     self.d, self.wa, self.ldc)
        for j, (r0, rc) in enumerate(ranges):
            if rc == 0:
                continue
            if self.fp8 and j == 1:
                rows = dict(batches=b, rows_per_batch=sl, row_begin=r0, row_count=rc)
                self.quant8(0, wa, r0, rc)
                with T("gemm_attn_out"):
                    ops.gemm_fp8(self.xn8[:, :, :wa], self.sc8, w["w_o"], w["s_o"], bo[j], PF_EPI_GATE_RESID, out=h, ldo=d,
                                 gate=mod[:, offs[j] + 2 * d:], gate_batch_stride=nm, **rows)
                self.ln8(offs[j] + 3 * d, offs[j] + 4 * d, r0, rc)
                with T("gemm_ff1_gelu"):
                    ops.gemm_fp8(self.xa8, self.sx8, w["w_f1"], w["s_f1"], bf1[j], PF_EPI_GELU_BF16, out=cat, ldo=ldc,
                                 out_col_begin=wa, **rows)
                self.quant8(wa, ldc, r0, rc)
                with T("gemm_ff2"):
                    ops.gemm_fp8(self.xn8[:, :, wa:], self.sc8, w["w_f2"], w["s_f2"], bf2[j], PF_EPI_GATE_RESID, out=h, ldo=d,
                                 gate=mod[:, offs[j] + 5 * d:], gate_batch_stride=nm, **rows)
                continue
            with T("gemm_attn_out"):
                ops.gemm(cat[:, :, :wa], wo[j], bo[j], PF_EPI_GATE_RESID, batches=b, rows_per_batch=sl, row_begin=r0,
                         row_count=rc, out=h, ldo=d, gate=mod[:, offs[j] + 2 * d:], gate_batch_stride=nm)   # gate_msa
            self.ln(offs[j] + 3 * d, offs[j] + 4 * d, r0, rc)                                     # (shift_mlp, scale_mlp)
            with T("gemm_ff1_gelu"):
                ops.gemm(xn, wf1[j], bf1[j], PF_EPI_GELU_BF16, batches=b, rows_per_batch=sl, row_begin=r0,
                         row_count=rc, out=cat, ldo=ldc, out_col_begin=wa)
            with T("gemm_ff2"):
                ops.gemm(cat[:, :, wa:], wf2[j], bf2[j], PF_EPI_GATE_RESID, batches=b, rows_per_batch=sl, row_begin=r0,
                         row_count=rc, out=h, ldo=d, gate=mod[:, offs[j] + 5 * d:], gate_batch_stride=nm)  # gate_mlp

    # ---- head: only the current clip's tokens are needed (F:380); AdaLN-continuous is (scale, shift) (N:119)
    def head(self) -> torch.Tensor:
        """proj_out of my rows among the last clip's tokens into the fp32 head [b, n_last, token_dim]; with the peer exchange
        every sp rank publishes its rows to every sp rank, so each holds all of them."""
        m, plan, c0, tw, d = self.m, self.plan, self.c0, self.m.token_dim, self.d
        n_last, s = plan.last_tokens, plan.seq
        o = m.mod_off["norm_out"]
        g0, g1 = max(s - n_last, c0), self.c1              # my part of the last n_last tokens
        peer = self.px is not None and self.nsp > 1
        head = self.px.head(n_last) if peer else self.ws["head"]
        if g1 > g0:
            self.ln(o + d, o, g0 - c0, g1 - g0)
            ops.gemm(self.xn, m.w_out, m.b_out, PF_EPI_STORE_F32, batches=self.b, rows_per_batch=self.sl, row_begin=g0 - c0,
                     row_count=g1 - g0, out=head, ldo=tw, out_batch_rows=n_last, out_row_begin=g0 - (s - n_last))
            if peer:
                r0h = g0 - (s - n_last)
                self.px.bcast(self.px.sp_buf, head[0, r0h:r0h + (g1 - g0)], self.px.off_head + r0h * tw * 4)
        if peer:
            self.px.barrier_sp()
        return head

    def unpatchify(self, head: torch.Tensor, clips) -> torch.Tensor:
        """The velocity of this rank's samples, in the clips' dtype (fp32 for other dtypes or with `output_fp32`)."""
        ct, chh, cww = self.plan.clip_thw[-1]
        odt = clips[-1].dtype if clips[-1].dtype in (torch.float32, torch.bfloat16) else torch.float32
        if self.m.output_fp32:
            odt = torch.float32
        out = torch.empty(self.b, self.m.token_dim // 4, ct, chh * 2, cww * 2, device=self.m.device, dtype=odt)
        ops.unpatchify(head, self.plan.last_tokens, 0, out)
        return out

    def publish(self, out: torch.Tensor) -> torch.Tensor:
        """With the peer exchange, the [uncond ; cond] velocity on every rank: the first sp rank of each branch publishes
        its velocity to every rank of the world."""
        px, lay = self.px, self.lay
        if px is None:
            return out
        vel = px.vel((self.bg, *out.shape[1:]), out.dtype)
        if lay.sp_rank == 0:
            px.bcast(px.world_buf, out.view(-1), px.w_off_vel + lay.cfg_rank * px.vel_bytes)
        px.barrier_world()
        return vel.clone()
