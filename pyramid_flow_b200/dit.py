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

Data layout in HBM (B = CFG batch, S = text + all clip tokens, D = heads*64):
  h    fp32 [B, S, D]      joint residual stream ([text ; clip_0 ; ... ; clip_n] per sample) — fp32 so that 48 residual
                           adds do not accumulate bf16 rounding (the reference keeps it bf16)
  xn   bf16 [B, S, D]      LN+modulated activations (GEMM A operand)
  q,k,v bf16 [B, H, S, 64] head-major, written by the QKV epilogue, read by TMA in the attention kernel
  cat  bf16 [B, S, 5D]     [attention out | MLP hidden] — proj_out of the single block reads it without a concat copy
  mod  fp32 [B, N_mod]     every layer's (shift, scale, gate, ...) from ONE GEMV per step
  fp8 only:
  xn8  e4m3 [B, S, 5D]     twin of `cat`: quantised [attention out | MLP hidden] rows; its first B*S*D bytes also hold the
                           LN-modulate output [B, S, D] (consumed by QKV / FF1 / proj_mlp before the twin is refilled)
  sx8, sc8 fp32 [B, S]     row scales of the LN-modulate output and of the quantised `cat` rows
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from . import _lib, ops
from ._lib import PF_EPI_GATE_RESID, PF_EPI_GELU_BF16, PF_EPI_QKV_ROPE, PF_EPI_STORE_F32
from .graphs import GraphedStep


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
    rope: torch.Tensor        # device fp32 [S, 32, 2]
    seg: torch.Tensor         # device int32 [B, S]
    time: torch.Tensor        # device int32 [B, S]
    sched: torch.Tensor       # device int32 [B, q_tiles, stride]
    sched2: object            # ops.PairSchedule on the device: pair schedule + row masks (pf_attn_build_pair_*)
    allowed_pairs: int        # sum over batch of allowed (q, kv) pairs (attention FLOP accounting)


def build_seq_plan(clip_shapes: Sequence[Sequence[int]], mask_cpu: torch.Tensor, axes_dim, patch: int, device) -> SeqPlan:
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


# ----------------------------------------------------------------------------------------------------------------------
# default formulation of the sequence-parallel exchange: "peer" (remote stores fused into the kernels over NVLink peer memory) once
# validated on hardware, else "nccl" (all_to_all_single)
DEFAULT_EXCHANGE = "peer"


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def check_gemm_precision(gemm_precision: str) -> None:
    if gemm_precision not in ("bf16", "fp8"):
        raise ValueError(f"gemm_precision must be 'bf16' or 'fp8', not {gemm_precision!r}")


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


class B200FluxTransformer(GraphedStep, torch.nn.Module):
    """Holder of packed bf16 weights + the kernel-launch sequence of one DiT step."""

    def __init__(self, config: FluxConfigB200, state_dict: Dict[str, torch.Tensor], device="cuda",
                 emulate_bf16_rounding: bool = False, gemm_precision: str = "bf16"):
        super().__init__()
        check_gemm_precision(gemm_precision)
        # "fp8": the block GEMMs listed in the module docstring run on e4m3 operands (opt-in: different numerics)
        self.gemm_precision = gemm_precision
        self.cfg = config
        # True reproduces the reference's bf16 rounding of the sinusoidal projection (E:195); False keeps fp32
        self.emulate_bf16_rounding = emulate_bf16_rounding
        self.config = _Cfg(in_channels=config.in_channels, num_layers=config.num_layers,
                           num_single_layers=config.num_single_layers,
                           num_attention_heads=config.num_attention_heads,
                           attention_head_dim=config.attention_head_dim,
                           joint_attention_dim=config.joint_attention_dim,
                           pooled_projection_dim=config.pooled_projection_dim)
        assert config.attention_head_dim == 64, "kernels are specialised for head_dim 64"
        self._plans: Dict[tuple, SeqPlan] = {}
        self._ws: Dict[tuple, dict] = {}
        self._import_state_dict(state_dict, torch.device(device))
        self.last_plan: Optional[SeqPlan] = None
        self._last_key = None
        self.attn_events = None   # bench.py: list collecting (start, end) CUDA events around every attention launch
        self.timer = _KernelTimer()
        self.trim_last_block = True     # last single block on the current clip's rows only (exact; see forward)
        self.attn_variant = 0           # pf_attn_desc.variant (every value runs the one sm_90a kernel)
        self._init_graphs()             # use_cuda_graph: the ~290 launches of a step captured once per shape (graphs.py)

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

    @property
    def device(self):
        return self.w_x.device

    @property
    def dtype(self):
        return torch.bfloat16

    def parameters(self, recurse: bool = True):  # the pipeline only asks next(self.dit.parameters()).device/.dtype
        return iter([self.w_x])

    # -- workspace -----------------------------------------------------------------------------------------------------
    def _workspace(self, b: int, plan: SeqPlan, sl: Optional[int] = None, hp: Optional[int] = None) -> dict:
        c = self.cfg
        sl = plan.seq if sl is None else sl
        hp = c.num_attention_heads if hp is None else hp
        key = (b, plan.seq, plan.video_len, plan.last_tokens, sl, hp)
        ws = self._ws.get(key)
        if ws is None:
            if len(self._ws) >= 4:   # shapes change every unit/stage; keep the cache bounded
                self._ws.clear()
            d, hn, dev = c.inner_dim, c.num_attention_heads, self.device
            alloc = torch.zeros if hp != hn else torch.empty      # padded heads must read as zeros
            ws = dict(
                h=torch.empty(b, sl, d, device=dev, dtype=torch.float32),
                xn=torch.empty(b, sl, d, device=dev, dtype=torch.bfloat16),
                q=alloc(b, hp, sl, 64, device=dev, dtype=torch.bfloat16),
                k=alloc(b, hp, sl, 64, device=dev, dtype=torch.bfloat16),
                v=alloc(b, hp, sl, 64, device=dev, dtype=torch.bfloat16),
                cat=torch.empty(b, sl, hp * 64 + 4 * d, device=dev, dtype=torch.bfloat16),
                tok=torch.empty(b, plan.video_len, c.in_channels, device=dev, dtype=torch.bfloat16),
                mod=torch.empty(b, self.n_mod, device=dev, dtype=torch.float32),
                temb=torch.empty(b, d, device=dev, dtype=torch.float32),
                tmp=torch.empty(b, d, device=dev, dtype=torch.float32),
                head=torch.zeros(b, plan.last_tokens, c.in_channels, device=dev, dtype=torch.float32),
            )
            if self.gemm_precision == "fp8":
                ws["xn8"] = torch.empty(b, sl, hp * 64 + 4 * d, device=dev, dtype=torch.float8_e4m3fn)
                ws["sx8"] = torch.empty(b, sl, device=dev, dtype=torch.float32)
                ws["sc8"] = torch.empty(b, sl, device=dev, dtype=torch.float32)
            if sl != plan.seq:   # sequence parallel: attention output of my head group over the whole sequence
                lay = self.layout
                ws["of"] = torch.empty(plan.seq, (hp // lay.sp) * 64, device=dev, dtype=torch.bfloat16)
            self._ws[key] = ws
        return ws

    def plan_for(self, clip_shapes, mask: torch.Tensor) -> SeqPlan:
        # fast path: the SAME mask tensor object (kept alive here, so its address cannot be recycled by the caching
        # allocator for a different mask), unmodified since, and the same clip shapes as the previous call -> no D2H sync
        shapes = tuple(tuple(int(x) for x in s) for s in clip_shapes)
        lk = self._last_key
        if lk is not None and lk[0] is mask and lk[1] == mask._version and lk[2] == shapes:
            return lk[3]
        plan = self._plan_slow(clip_shapes, mask)
        self._last_key = (mask, mask._version, shapes, plan)
        return plan

    def _plan_slow(self, clip_shapes, mask: torch.Tensor) -> SeqPlan:
        mask_cpu = mask.detach().to("cpu", torch.int64)
        key = (tuple(tuple(int(x) for x in s) for s in clip_shapes), mask_cpu.shape, bytes(mask_cpu.numpy().tobytes()))
        plan = self._plans.get(key)
        if plan is None:
            if len(self._plans) >= 16:
                self._plans.clear()
            plan = build_seq_plan(clip_shapes, mask_cpu, self.cfg.axes_dims_rope, self.cfg.patch_size, self.device)
            self._plans[key] = plan
        return plan

    # -- parallel layout (CFG x sequence parallel, sp.py) ---------------------------------------------------------------
    def set_parallel_layout(self, layout, exchange: str = DEFAULT_EXCHANGE) -> None:
        """Attach a `sp.ParallelLayout` (after torch.distributed is initialised); weights are replicated.
        exchange = "peer": q/k/v and the attention output cross NVLink as remote stores fused into the QKV GEMM / attention
        epilogues + flag barriers (csrc/pf_peer.cu): no NCCL call in the step, CUDA-graph capturable.  "nccl": the
        all_to_all_single formulation (kept for A/B measurements)."""
        if self.gemm_precision == "fp8":
            raise NotImplementedError("gemm_precision='fp8' runs on one GPU only: the sequence-parallel peer-store epilogues "
                                      "have no fp8 form (build the model with gemm_precision='bf16' for a parallel layout)")
        assert exchange in ("peer", "nccl")
        if layout.sp > 1:   # see _lib.load(): one attention kernel for the whole process once sequence parallelism is in play
            _lib.set_option(_lib.PF_OPT_ATTN_TRIPLE_KERNEL, 0)
        self.layout = layout
        self.exchange = exchange
        self._px = None
        self._graphs.clear()
        self._ws.clear()
        hn = self.cfg.num_attention_heads
        from .sp import padded_heads
        hp = padded_heads(hn, layout.sp)
        self._hp = hp
        if hp != hn and not hasattr(self, "_padded"):
            d, pad = self.cfg.inner_dim, (hp - hn) * 64

            def padk(w):   # [N, D (+rest)] -> [N, Hp*64 (+rest)]: zero columns for the padded heads
                z = torch.zeros(w.shape[0], pad, device=w.device, dtype=w.dtype)
                return torch.cat([w[:, :d], z, w[:, d:]], dim=1).contiguous()

            for blk in self.dbl:
                blk["w_o_p"], blk["w_co_p"] = padk(blk["w_o"]), padk(blk["w_co"])
            for blk in self.sgl:
                blk["w_out_p"] = padk(blk["w_out"])
            self._padded = True

    def _peer_exchange(self, plan: SeqPlan, hp: int, ldc: int):
        """The peer arena (sp.PeerExchange) for this call's shapes; see sp.ensure_peer_exchange."""
        from . import sp as SP
        c = self.cfg
        ct, chh, cww = plan.clip_thw[-1]
        vel_bytes = (c.in_channels // 4) * ct * chh * 2 * cww * 2 * 4
        return SP.ensure_peer_exchange(self, self.layout, plan.seq, plan.last_tokens, hp, ldc, c.in_channels, vel_bytes)

    # -- the step ------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, sample, timestep_ratio=None, encoder_hidden_states=None, encoder_attention_mask=None,
                pooled_projections=None):
        _lib.require_device()
        assert len(sample) == 1, "inference passes one stage per call (pipeline P:760-766)"
        clips = sample[0] if isinstance(sample[0], (list, tuple)) else [sample[0]]
        lay = getattr(self, "layout", None)
        # the NCCL formulation of the parallel step stays host-launched (its all-to-alls are not captured); the peer-memory formulation is plain kernels and is captured like the single-GPU step
        nccl_par = lay is not None and lay.enabled and getattr(self, "exchange", DEFAULT_EXCHANGE) == "nccl"
        if self.use_cuda_graph and not nccl_par and not self.timer.enabled and self.attn_events is None:
            return self._forward_graphed(list(clips), timestep_ratio, encoder_hidden_states, encoder_attention_mask,
                                         pooled_projections)
        return self._forward_eager(clips, timestep_ratio, encoder_hidden_states, encoder_attention_mask,
                                   pooled_projections)

    # -- CUDA-graph replay (graphs.GraphedStep) -------------------------------------------------------------------------
    def _graph_key_fields(self) -> tuple:
        return (bool(getattr(self, "output_fp32", False)), bool(self.trim_last_block), bool(self.emulate_bf16_rounding),
                int(self.attn_variant))

    def _graph_prealloc(self, plan: SeqPlan, clips) -> None:
        lay = getattr(self, "layout", None)
        if lay is not None and lay.enabled:
            from . import sp as SP
            c0, c1 = SP.chunk_bounds(plan.seq, lay.sp, lay.sp_rank)
            self._workspace(1, plan, c1 - c0, self._hp)
            if getattr(self, "exchange", DEFAULT_EXCHANGE) == "peer":
                self._peer_exchange(plan, self._hp, self._hp * 64 + 4 * self.cfg.inner_dim)
        else:
            self._workspace(clips[-1].shape[0], plan)

    def _forward_eager(self, clips, timestep_ratio=None, encoder_hidden_states=None, encoder_attention_mask=None,
                       pooled_projections=None):
        c = self.cfg
        d, hn = c.inner_dim, c.num_attention_heads
        lay = getattr(self, "layout", None)
        par = lay is not None and lay.enabled
        bg = clips[-1].shape[0]                       # global (CFG) batch
        plan = self.plan_for([cl.shape for cl in clips], encoder_attention_mask)
        self.last_plan = plan
        t_len, s, lv = plan.text_len, plan.seq, plan.video_len
        if par:
            from . import sp as SP
            assert bg == lay.cfg_ways, "CFG-parallel layout expects the [uncond ; cond] batch"
            b, b0 = 1, lay.cfg_rank                    # this rank's CFG branch
            nsp, hp = lay.sp, self._hp
            c0, c1 = SP.chunk_bounds(s, nsp, lay.sp_rank)
        else:
            b, b0, nsp, hp, c0, c1 = bg, 0, 1, hn, 0, s
        sl = c1 - c0                                   # tokens of the joint sequence owned by this rank
        wa = hp * 64                                   # width of the attention block in `cat`
        ws = self._workspace(b, plan, sl, hp)
        h, xn, q, k, v, cat, mod = ws["h"], ws["xn"], ws["q"], ws["k"], ws["v"], ws["cat"], ws["mod"]
        nm = self.n_mod
        ldc = wa + 4 * d
        # peer-memory formulation of the exchanges (sp.PeerExchange): `cat` and the gathered q/k/v live in the peer arena
        px = self._peer_exchange(plan, hp, ldc) if (par and getattr(self, "exchange", DEFAULT_EXCHANGE) == "peer") else None
        if px is not None and nsp > 1:
            cat = px.cat(sl)
            qkv_x = px.qkv(s)                          # [3, Hg, S, 64]: my head group over the whole sequence
        rope = plan.rope[c0:c1]
        # local (row_begin, row_count) of the text / video ranges inside this rank's chunk, and their global starts
        tb, te = max(0, c0), min(t_len, c1)
        vb, ve = max(t_len, c0), min(s, c1)
        ranges = ((tb - c0, max(0, te - tb)), (vb - c0, max(0, ve - vb)))

        # ---- conditioning (E:193-201): timestep arrives already rounded to bf16 by the pipeline (P:750)
        t32 = timestep_ratio.detach().to(device=self.device, dtype=torch.float32)[b0:b0 + b].contiguous()
        tproj = ops.timestep_embedding(t32, 256, round_bf16=self.emulate_bf16_rounding)
        ops.small_linear(tproj, self.w_t1, self.b_t1, ws["tmp"], act_out=1)
        ops.small_linear(ws["tmp"], self.w_t2, self.b_t2, ws["temb"])
        pooled = pooled_projections.detach().to(device=self.device, dtype=torch.float32)[b0:b0 + b].contiguous()
        ops.small_linear(pooled, self.w_p1, self.b_p1, ws["tmp"], act_out=1)
        ops.small_linear(ws["tmp"], self.w_p2, self.b_p2, ws["temb"], accumulate=True)
        # ---- every AdaLN modulation of the step in one GEMV: mod = Linear(SiLU(temb)) for all layers
        ops.small_linear(ws["temb"], self.w_mod, self.b_mod, mod, act_in=1)

        # ---- embedders write straight into the joint fp32 residual stream (only this rank's rows)
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
            ops.gemm(ws["tok"], self.w_x, self.b_x, PF_EPI_STORE_F32, batches=b, rows_per_batch=lv, row_begin=vb - t_len,
                     row_count=ve - vb, out=h, ldo=d, out_batch_rows=sl, out_row_begin=vb - c0)

        T = self.timer

        def lnmod(off_shift, off_scale, r0, rc):
            if rc > 0:
                with T("ln_modulate"):
                    ops.ln_modulate(h, xn, mod[:, off_shift:], mod[:, off_scale:], nm, batches=b, rows_per_batch=sl,
                                    row_begin=r0, row_count=rc)

        fp8 = self.gemm_precision == "fp8"
        if fp8:
            xn8, sx8, sc8 = ws["xn8"], ws["sx8"], ws["sc8"]
            xa8 = xn8.view(-1)[:b * sl * d].view(b, sl, d)    # LN-modulate output, row stride d (module docstring)

        def lnmod8(off_shift, off_scale, r0, rc):
            with T("ln_modulate"):
                ops.ln_modulate_fp8(h, xa8, sx8, mod[:, off_shift:], mod[:, off_scale:], nm, batches=b, rows_per_batch=sl,
                                    row_begin=r0, row_count=rc)

        def quant8(col0, col1, r0, rc):   # cat[:, r0:r0 + rc, col0:col1] -> the same block of xn8, row scales -> sc8
            with T("quantize_fp8"):
                ops.quantize_rows_fp8(cat[:, :, col0:col1], xn8[:, :, col0:col1], sc8, batches=b, rows_per_batch=sl,
                                      row_begin=r0, row_count=rc)

        peer_qkv = None
        if px is not None and nsp > 1:
            # QKV epilogue stores head h of my rows into rank (h // Hg)'s gathered buffer at sequence position c0 + row
            peer_qkv = dict(peer_ptrs=[pp + px.off_qkv for pp in px.sp_buf.ptrs], peer_heads=hp // nsp, peer_seq=s, peer_row0=c0)

        def qkv(wq, bq, nq, nk, r0, rc):
            if rc > 0:
                with T("gemm_qkv"):
                    ops.gemm(xn, wq, bq, PF_EPI_QKV_ROPE, batches=b, rows_per_batch=sl, row_begin=r0, row_count=rc,
                             q_out=q, k_out=k, v_out=v, rope=rope, q_norm_w=nq, k_norm_w=nk, heads=hn, head_dim=64,
                             seq_len=sl, peer=peer_qkv)

        def qkv8(wq, sq, bq, nq, nk, r0, rc):
            with T("gemm_qkv"):
                ops.gemm_fp8(xa8, sx8, wq, sq, bq, PF_EPI_QKV_ROPE, batches=b, rows_per_batch=sl, row_begin=r0, row_count=rc,
                             q_out=q, k_out=k, v_out=v, rope=rope, q_norm_w=nq, k_norm_w=nk, heads=hn, head_dim=64,
                             seq_len=sl)

        scale = 1.0 / math.sqrt(64)
        seg, tim, sched, sched2 = plan.seg[b0:b0 + b], plan.time[b0:b0 + b], plan.sched[b0:b0 + b], plan.sched2[b0:b0 + b]
        av = self.attn_variant

        def exchange_begin():
            if nsp > 1 and px is None:
                return SP.heads_to_sequence_qkv_begin(q[0], k[0], v[0], lay)
            return None

        def attention(pending=None, q_row_begin=0):
            ev = self.attn_events is not None
            if ev:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            if nsp == 1:
                if ev:
                    e0.record()
                ops.attn_fwd(q, k, v, cat, seg, tim, sched, scale, variant=av, q_row_begin=q_row_begin, pair_sched=sched2)
                if ev:
                    e1.record()
            elif px is not None:
                # every rank's QKV epilogue has stored into every rank's gathered buffer: order those stores before the reads;
                # the attention epilogue then stores each token chunk's rows straight into its owner's `cat`; the second
                # barrier orders those stores before the projections that read `cat`
                px.barrier_sp()
                if ev:
                    e0.record()
                ops.attn_fwd(qkv_x[0][None], qkv_x[1][None], qkv_x[2][None], None, seg, tim, sched, scale, variant=av,
                             pair_sched=sched2, ldo=ldc,
                             peer=dict(peer_ptrs=[pp + px.off_cat for pp in px.sp_buf.ptrs], peer_chunk_rows=sl,
                                       peer_col_begin=lay.sp_rank * (hp // nsp) * 64))
                if ev:
                    e1.record()
                px.barrier_sp()
            else:
                # Ulysses exchange: all (padded) heads of my token chunk -> my head group over the whole sequence
                qf, kf, vf = SP.heads_to_sequence_qkv_end(pending if pending is not None else exchange_begin())
                of = ws["of"]
                if ev:
                    e0.record()
                ops.attn_fwd(qf[None], kf[None], vf[None], of[None], seg, tim, sched, scale, variant=av, pair_sched=sched2)
                if ev:
                    e1.record()
                cat[0, :, :wa].copy_(SP.sequence_to_heads(of, lay))
            if ev:
                self.attn_events.append((e0, e1))

        pad = hp != hn
        for i, w in enumerate(self.dbl):
            ov = self.mod_off[f"transformer_blocks.{i}.norm1"]
            oc = self.mod_off[f"transformer_blocks.{i}.norm1_context"]
            offs = (oc, ov)
            wq, bq, nq, nk = (w["w_cqkv"], w["w_qkv"]), (w["b_cqkv"], w["b_qkv"]), (w["cnq"], w["nq"]), (w["cnk"], w["nk"])
            wo = (w["w_co_p"], w["w_o_p"]) if pad else (w["w_co"], w["w_o"])
            bo = (w["b_co"], w["b_o"])
            wf1, bf1 = (w["w_cf1"], w["w_f1"]), (w["b_cf1"], w["b_f1"])
            wf2, bf2 = (w["w_cf2"], w["w_f2"]), (w["b_cf2"], w["b_f2"])
            for j, (r0, rc) in enumerate(ranges):
                if fp8 and j == 1 and rc > 0:                              # video range in fp8
                    lnmod8(offs[j] + 0 * d, offs[j] + 1 * d, r0, rc)
                    qkv8(w["w_qkv"], w["s_qkv"], bq[j], nq[j], nk[j], r0, rc)
                    continue
                lnmod(offs[j] + 0 * d, offs[j] + 1 * d, r0, rc)            # (shift_msa, scale_msa) N:173/191
                qkv(wq[j], bq[j], nq[j], nk[j], r0, rc)
            attention()
            for j, (r0, rc) in enumerate(ranges):
                if rc == 0:
                    continue
                if fp8 and j == 1:
                    rows = dict(batches=b, rows_per_batch=sl, row_begin=r0, row_count=rc)
                    quant8(0, wa, r0, rc)
                    with T("gemm_attn_out"):
                        ops.gemm_fp8(xn8[:, :, :wa], sc8, w["w_o"], w["s_o"], bo[j], PF_EPI_GATE_RESID, out=h, ldo=d,
                                     gate=mod[:, offs[j] + 2 * d:], gate_batch_stride=nm, **rows)
                    lnmod8(offs[j] + 3 * d, offs[j] + 4 * d, r0, rc)
                    with T("gemm_ff1_gelu"):
                        ops.gemm_fp8(xa8, sx8, w["w_f1"], w["s_f1"], bf1[j], PF_EPI_GELU_BF16, out=cat, ldo=ldc,
                                     out_col_begin=wa, **rows)
                    quant8(wa, ldc, r0, rc)
                    with T("gemm_ff2"):
                        ops.gemm_fp8(xn8[:, :, wa:], sc8, w["w_f2"], w["s_f2"], bf2[j], PF_EPI_GATE_RESID, out=h, ldo=d,
                                     gate=mod[:, offs[j] + 5 * d:], gate_batch_stride=nm, **rows)
                    continue
                with T("gemm_attn_out"):
                    ops.gemm(cat[:, :, :wa], wo[j], bo[j], PF_EPI_GATE_RESID, batches=b, rows_per_batch=sl, row_begin=r0,
                             row_count=rc, out=h, ldo=d, gate=mod[:, offs[j] + 2 * d:], gate_batch_stride=nm)   # gate_msa
                lnmod(offs[j] + 3 * d, offs[j] + 4 * d, r0, rc)                                   # (shift_mlp, scale_mlp)
                with T("gemm_ff1_gelu"):
                    ops.gemm(xn, wf1[j], bf1[j], PF_EPI_GELU_BF16, batches=b, rows_per_batch=sl, row_begin=r0,
                             row_count=rc, out=cat, ldo=ldc, out_col_begin=wa)
                with T("gemm_ff2"):
                    ops.gemm(cat[:, :, wa:], wf2[j], bf2[j], PF_EPI_GATE_RESID, batches=b, rows_per_batch=sl, row_begin=r0,
                             row_count=rc, out=h, ldo=d, gate=mod[:, offs[j] + 5 * d:], gate_batch_stride=nm)  # gate_mlp

        n_last = plan.last_tokens
        for i, w in enumerate(self.sgl):
            o = self.mod_off[f"single_transformer_blocks.{i}.norm"]
            # Last block: only the current clip's tokens are read afterwards (F:380), so its queries, MLP and projection
            # run on the rows from the 128-aligned start of the current clip; K/V still cover every token.  Same kernels
            # on fewer rows: the kept rows are bit-identical.  (Single-GPU layout; SP chunks stay uniform.)
            r0 = ((s - n_last) // 128) * 128 if (self.trim_last_block and not par and i == len(self.sgl) - 1) else 0
            if fp8:
                rows = dict(batches=b, rows_per_batch=sl, row_begin=r0, row_count=sl - r0)
                lnmod8(o, o + d, 0, sl)
                qkv8(w["w_qkv"], w["s_qkv"], w["b_qkv"], w["nq"], w["nk"], 0, sl)
                with T("gemm_single_mlp_gelu"):
                    ops.gemm_fp8(xa8, sx8, w["w_mlp"], w["s_mlp"], w["b_mlp"], PF_EPI_GELU_BF16, out=cat, ldo=ldc,
                                 out_col_begin=wa, **rows)
                attention(q_row_begin=r0)
                quant8(0, ldc, r0, sl - r0)
                with T("gemm_single_out"):
                    ops.gemm_fp8(xn8, sc8, w["w_out"], w["s_out"], w["b_out"], PF_EPI_GATE_RESID, out=h, ldo=d,
                                 gate=mod[:, o + 2 * d:], gate_batch_stride=nm, **rows)
                continue
            lnmod(o, o + d, 0, sl)                                                                 # (shift, scale) N:232
            # two launches sharing A: measured faster than the fused q|k|v|mlp GEMM (PF_EPI_QKV_GELU), whose 192-wide
            # tiles slow the MLP half down (1.81 ms fused vs 0.60 + 0.62 ms split at S=15488)
            qkv(w["w_qkv"], w["b_qkv"], w["nq"], w["nk"], 0, sl)
            pending = exchange_begin()       # SP: the q/k/v all-to-alls run under the proj_mlp GEMM
            with T("gemm_single_mlp_gelu"):
                ops.gemm(xn, w["w_mlp"], w["b_mlp"], PF_EPI_GELU_BF16, batches=b, rows_per_batch=sl, row_begin=r0,
                         row_count=sl - r0, out=cat, ldo=ldc, out_col_begin=wa)
            attention(pending, q_row_begin=r0)
            with T("gemm_single_out"):
                ops.gemm(cat, w["w_out_p"] if pad else w["w_out"], w["b_out"], PF_EPI_GATE_RESID, batches=b,
                         rows_per_batch=sl, row_begin=r0, row_count=sl - r0, out=h, ldo=d, gate=mod[:, o + 2 * d:],
                         gate_batch_stride=nm)

        # ---- head: only the current clip's tokens are needed (F:380); AdaLN-continuous is (scale, shift) (N:119)
        o = self.mod_off["norm_out"]
        g0, g1 = max(s - n_last, c0), c1                 # my part of the last n_last tokens
        head = ws["head"]
        peer_head = px is not None and nsp > 1
        if peer_head:
            head = px.head(n_last)                    # peer arena: every sp rank publishes its rows to every sp rank
        elif par and nsp > 1:
            head.zero_()
        if g1 > g0:
            lnmod(o + d, o, g0 - c0, g1 - g0)
            ops.gemm(xn, self.w_out, self.b_out, PF_EPI_STORE_F32, batches=b, rows_per_batch=sl, row_begin=g0 - c0,
                     row_count=g1 - g0, out=head, ldo=c.in_channels, out_batch_rows=n_last,
                     out_row_begin=g0 - (s - n_last))
            if peer_head:
                r0h = g0 - (s - n_last)
                px.bcast(px.sp_buf, head[0, r0h:r0h + (g1 - g0)], px.off_head + r0h * c.in_channels * 4)
        if peer_head:
            px.barrier_sp()
        elif par and nsp > 1:
            torch.distributed.all_reduce(head, group=lay.sp_group)       # disjoint row blocks: sum == gather
        ct, chh, cww = plan.clip_thw[-1]
        odt = clips[-1].dtype if clips[-1].dtype in (torch.float32, torch.bfloat16) else torch.float32
        if getattr(self, "output_fp32", False):       # fused CFG+Euler path of the sampler keeps the velocity in fp32
            odt = torch.float32
        out = torch.empty(b, c.in_channels // 4, ct, chh * 2, cww * 2, device=self.device, dtype=odt)
        ops.unpatchify(head, n_last, 0, out)
        if par and px is not None:
            # [uncond ; cond]: the first sp rank of each branch publishes its velocity to every rank of the world
            vel = px.vel((bg, *out.shape[1:]), odt)
            if lay.sp_rank == 0:
                px.bcast(px.world_buf, out.view(-1), px.w_off_vel + lay.cfg_rank * px.vel_bytes)
            px.barrier_world()
            out = vel.clone()
        elif par:
            full = torch.empty(bg, *out.shape[1:], device=self.device, dtype=odt)
            torch.distributed.all_gather_into_tensor(full, out, group=lay.cfg_group)   # [uncond ; cond]
            out = full
        return [out]

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
