"""Trainable masked attention, and its drop-in for the reference's autoregressive training path.

`masked_attention(q, k, v, seg, time, scale)` is softmax attention under mask(q, kv) = (seg[q] == seg[kv]) &&
(time[q] >= time[kv]) with a backward: the forward is pf_attn_fwd_masked (which also stores each row's log-sum-exp), the
backward pf_attn_bwd_masked (include/pf_b200.h).  Gradients are taken w.r.t. the bf16 q / k / v with fp32 accumulation, and are
deterministic (no atomics), so a forward recomputed under torch.utils.checkpoint gives the bits of the first one.

`install_training_attention(ref_dit)` puts it under an unmodified reference `PyramidFluxTransformer` or
`PyramidDiffusionMMDiT` instance, trained with `use_flash_attn=False` (scripts/train_pyramid_flow.sh without
--use_flash_attn): the `varlen_attn` callable of every FluxAttnProcessor2_0 / FluxSingleAttnProcessor2_0
(VarlenSelfAttentionWithT5Mask B:328-376, VarlenSelfAttnSingle B:568-606), or the `var_len_attn` of every MMDiT
JointAttention (VarlenSelfAttentionWithT5Mask MB:262-322, the last, context_pre_only block included), is replaced by a library
callable with the same signature and output layout, and the instance's `merge_input` (F:239-352, M:265-380) is wrapped so
that each stage's dense [B, 1, S, S] bool mask (F:341-350, M:369-378) becomes a `StageAttentionPlan` carrying that stage's
seg / time ids and tile schedules.  No reference source changes; `uninstall_training_attention` restores the instance.

At each call site the stacking of q / k / v, the concatenation of a stage's text rows with its video rows, the reference's
fp32 apply_rope and the head-major transpose run as one kernel per stage (pf_attn_stage_pack), with the same bits as that
torch code; its backward (pf_attn_stage_pack_bwd) writes the source gradients autograd would compute through it.

`install_varlen_training_attention(ref_dit)` does the same for a PyramidFluxTransformer built with use_flash_attn=True
(scripts/train_pyramid_flow_without_ar.sh): every processor's `varlen_flash_attn` (VarlenFlashSelfAttentionWithT5Mask
B:189-263, VarlenFlashSelfAttnSingle B:452-516) is replaced, and merge_input's per-stage `indices` / `seqlens_in_batch`
(F:295-317) become one `VarlenAttentionPlan`.  Each call site then runs three launches forward, every stage at once and without
the padded text rows: pf_attn_varlen_pack (stack / cat / apply_rope / index_first_axis / cat), pf_attn_fwd_masked over the
packed sequences, pf_attn_varlen_unpack (pad_input into zeros).  `varlen_attention` is the flash_attn_varlen_func subset
the reference calls, on the same kernels.  The flash_attn package is not needed.
"""
from __future__ import annotations

import sys
from typing import Dict, Optional, Tuple

import torch

from . import _lib, ops

HEAD_DIM = 64


class StageAttentionPlan:
    """One stage's attention mask in the form the kernels take: seg / time int32 [B, S] on the device, the q-tile schedule
    (pf_attn_build_schedule) and its kv-major transpose (pf_attn_build_kv_schedule), both on the device."""

    def __init__(self, seg: torch.Tensor, time: torch.Tensor, sched: torch.Tensor, kv_sched: torch.Tensor):
        self.seg, self.time, self.sched, self.kv_sched = seg, time, sched, kv_sched

    @property
    def shape(self) -> Tuple[int, int]:
        return tuple(self.seg.shape)


_PLANS: Dict[tuple, StageAttentionPlan] = {}
_PLAN_CACHE_SIZE = 32


def plan_for(seg: torch.Tensor, time: torch.Tensor, device=None) -> StageAttentionPlan:
    """The StageAttentionPlan of seg / time ids [B, S] (any integer dtype, any device), cached by their content: a training
    run sees a handful of stage layouts, so after the first steps this costs one small device-to-host copy."""
    device = torch.device(device) if device is not None else seg.device
    seg_c = seg.detach().to("cpu", torch.int32).contiguous()
    time_c = time.detach().to("cpu", torch.int32).contiguous()
    assert seg_c.ndim == 2 and seg_c.shape == time_c.shape, (seg_c.shape, time_c.shape)
    key = (str(device), tuple(seg_c.shape), seg_c.numpy().tobytes(), time_c.numpy().tobytes())
    plan = _PLANS.get(key)
    if plan is None:
        sched, _ = ops.attn_build_schedule(seg_c, time_c)
        kv_sched = ops.attn_build_kv_schedule(sched, seg_c.shape[1])
        plan = StageAttentionPlan(seg_c.to(device), time_c.to(device), sched.to(device), kv_sched.to(device))
        if len(_PLANS) >= _PLAN_CACHE_SIZE:
            _PLANS.clear()
        _PLANS[key] = plan
    return plan


class _MaskedAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, plan: StageAttentionPlan, scale: float):
        b, h, s, hd = q.shape
        out = torch.empty(b, s, h * hd, dtype=torch.bfloat16, device=q.device)
        lse = torch.empty(b, h, s, dtype=torch.float32, device=q.device)
        ops.attn_fwd(q, k, v, out, plan.seg, plan.time, plan.sched, scale, lse=lse)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.plan, ctx.scale = plan, scale
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse = ctx.saved_tensors
        plan = ctx.plan
        dout = dout.to(torch.bfloat16)
        # a stage's slice of a wider gradient (the single blocks' cat along the sequence, then with the MLP branch) arrives
        # as a view with its own row and batch strides: passed as they are when the kernels can address them
        if not ops.attn_bwd_rows_ok(dout):
            dout = dout.contiguous()
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        ops.attn_bwd(q, k, v, out, dout, lse, plan.seg, plan.time, plan.sched, plan.kv_sched, ctx.scale, dq, dk, dv)
        return dq, dk, dv, None, None


def _check_qkv(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor) -> None:
    if q.shape[-1] != HEAD_DIM:
        raise ValueError(f"masked_attention: head_dim {q.shape[-1]} unsupported (the kernels are written for {HEAD_DIM})")
    if not (q.shape == k.shape == v.shape) or q.ndim != 4:
        raise ValueError(f"masked_attention: q, k, v must all be [B, H, S, {HEAD_DIM}] (got {q.shape}, {k.shape}, {v.shape})")
    if not q.is_cuda:
        raise RuntimeError("masked_attention runs on the GPU only (pyramid_flow_b200 has no CPU path)")


def attend(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, plan: StageAttentionPlan, scale: float) -> torch.Tensor:
    """q, k, v [B, H, S, 64] (any float dtype; taken to bf16) -> out [B, S, H*64] in q's dtype, under the plan's mask."""
    _check_qkv(q, k, v)
    if tuple(plan.shape) != (q.shape[0], q.shape[2]):
        raise ValueError(f"masked_attention: plan is for [B, S] = {tuple(plan.shape)}, q is {tuple(q.shape)}")
    _lib.require_device()
    dt = q.dtype
    q, k, v = (t.to(torch.bfloat16).contiguous() for t in (q, k, v))
    out = _MaskedAttention.apply(q, k, v, plan, float(scale))
    return out if dt == torch.bfloat16 else out.to(dt)


def masked_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, seg: torch.Tensor, time: torch.Tensor,
                     scale: Optional[float] = None) -> torch.Tensor:
    """softmax(q k^T * scale | mask) v with mask(i, j) = (seg[b, i] == seg[b, j]) && (time[b, i] >= time[b, j]), differentiable
    w.r.t. q, k, v.  q, k, v: [B, H, S, 64]; seg / time: integer [B, S]; scale defaults to 64 ** -0.5 (SDPA's default).
    Returns [B, S, H*64] (the layout SDPA's output takes after .transpose(1, 2).flatten(2, 3))."""
    _check_qkv(q, k, v)
    scale = q.shape[-1] ** -0.5 if scale is None else scale
    return attend(q, k, v, plan_for(seg, time, q.device), scale)


# ----------------------------------------------------------------------------------------------------------------------
# drop-in for the reference training path
# ----------------------------------------------------------------------------------------------------------------------
def _stage_plan(attention_mask, i_p: int) -> StageAttentionPlan:
    plan = attention_mask[i_p] if attention_mask is not None else None
    if not isinstance(plan, StageAttentionPlan):
        raise TypeError("the installed training attention takes the StageAttentionPlan objects of the wrapped merge_input, "
                        f"got {type(plan).__name__} (was the model's merge_input replaced after install_training_attention?)")
    return plan


class _StagePack(torch.autograd.Function):
    """Every stage of one call site packed into the kernels' head-major q / k / v (pf_attn_stage_pack, RoPE included).  The
    forward packs all stages so that the backward (pf_attn_stage_pack_bwd per stage) writes each row of each source gradient
    exactly once: no accumulation, and nothing of the sources is kept for the backward (only the RoPE tables)."""

    @staticmethod
    def forward(ctx, hidden_length, has_text: bool, *tensors):
        n = len(hidden_length)
        video = tensors[:3]
        text = tensors[3:6] if has_text else None
        freqs = tensors[6 if has_text else 3:] or None
        text_len = text[0].shape[1] if text is not None else 0
        b, _, h, hd = video[0].shape
        packed, row0 = [], 0
        for i_p, length in enumerate(hidden_length):
            stage = tuple(torch.empty(b, h, text_len + length, hd, dtype=torch.bfloat16, device=video[0].device) for _ in range(3))
            ops.attn_stage_pack(video, text, None if freqs is None else freqs[i_p], stage, row0=row0, stage=i_p, n_stages=n)
            packed += stage
            row0 += length
        ctx.hidden_length, ctx.has_text = list(hidden_length), has_text
        ctx.sources = [(t.shape, t.dtype) for t in tensors[:6 if has_text else 3]]
        if freqs is not None:
            ctx.save_for_backward(*freqs)
        return tuple(packed)

    @staticmethod
    def backward(ctx, *grads):
        freqs = ctx.saved_tensors or None
        dev = grads[0].device
        dsrc = [torch.empty(shape, dtype=dt, device=dev) for shape, dt in ctx.sources]
        dvideo, dtext = tuple(dsrc[:3]), (tuple(dsrc[3:]) if ctx.has_text else None)
        n, row0 = len(ctx.hidden_length), 0
        for i_p, length in enumerate(ctx.hidden_length):
            g = tuple(t.contiguous() for t in grads[3 * i_p:3 * i_p + 3])
            ops.attn_stage_pack_bwd(dvideo, dtext, None if freqs is None else freqs[i_p], g, row0=row0, stage=i_p, n_stages=n)
            row0 += length
        return (None, None, *dsrc) + (None,) * (0 if freqs is None else len(freqs))


def _attend_stages(video, text, hidden_length, image_rotary_emb, attention_mask) -> list:
    """The call site's attention, stage by stage: per stage i_p its text rows (encoder rows i_p::stages, when `text` is given)
    then its video rows, the reference's apply_rope with image_rotary_emb[i_p], attention under the stage's plan.  Returns each
    stage's output [B, T + L, H*64] in the dtype the reference's torch.stack / torch.cat of the sources gives."""
    sources = tuple(video) + (tuple(text) if text is not None else ())
    for t in sources:
        if t.ndim != 4 or t.shape[-1] != HEAD_DIM:
            raise ValueError(f"training attention: q / k / v must be [B, S, H, {HEAD_DIM}] (got {tuple(t.shape)})")
        if t.dtype not in (torch.bfloat16, torch.float32):
            raise ValueError(f"training attention: q / k / v must be bf16 or fp32 (got {t.dtype})")
    b, s_total = video[0].shape[:2]
    if sum(hidden_length) != s_total or (text is not None and text[0].shape[0] != b * len(hidden_length)):
        raise ValueError(f"training attention: stages {list(hidden_length)} do not cover the sources "
                         f"({tuple(video[0].shape)}{'' if text is None else f', text {tuple(text[0].shape)}'})")
    if not video[0].is_cuda:
        raise RuntimeError("masked_attention runs on the GPU only (pyramid_flow_b200 has no CPU path)")
    _lib.require_device()
    plans = [_stage_plan(attention_mask, i_p) for i_p in range(len(hidden_length))]
    text_len = text[0].shape[1] if text is not None else 0
    for plan, length in zip(plans, hidden_length):
        if tuple(plan.shape) != (b, text_len + length):
            raise ValueError(f"masked_attention: plan is for [B, S] = {tuple(plan.shape)}, the stage is {(b, text_len + length)}")
    dt = sources[0].dtype
    for t in sources[1:]:
        dt = torch.promote_types(dt, t.dtype)
    sources = tuple(t if ops.attn_pack_source_ok(t) else t.contiguous() for t in sources)
    freqs = tuple(image_rotary_emb[i_p] for i_p in range(len(hidden_length))) if image_rotary_emb is not None else ()
    packed = _StagePack.apply(list(hidden_length), text is not None, *sources, *freqs)
    outs = []
    for i_p, plan in enumerate(plans):
        q, k, v = packed[3 * i_p:3 * i_p + 3]
        out = _MaskedAttention.apply(q, k, v, plan, HEAD_DIM ** -0.5)
        outs.append(out if dt == torch.bfloat16 else out.to(dt))
    return outs


class _JointAttention:
    """Stands for VarlenSelfAttentionWithT5Mask (B:328-376, MB:262-322): per stage, text tokens of that stage (encoder rows
    i_p::stages) then its video tokens; the reference's apply_rope; attention under the stage's plan; outputs split back."""

    def __call__(self, query, key, value, encoder_query, encoder_key, encoder_value, heads, scale, hidden_length=None,
                 image_rotary_emb=None, attention_mask=None):
        encoder_length = encoder_query.shape[1]
        outs = _attend_stages((query, key, value), (encoder_query, encoder_key, encoder_value), hidden_length,
                              image_rotary_emb, attention_mask)
        # 'b n s d -> (b n) s d'
        return (torch.cat([o[:, encoder_length:] for o in outs], dim=1),
                torch.stack([o[:, :encoder_length] for o in outs], dim=1).flatten(0, 1))


class _SingleAttention:
    """Stands for VarlenSelfAttnSingle (B:568-606): the single blocks' joint sequence is already stage-major."""

    def __call__(self, query, key, value, heads, scale, hidden_length=None, image_rotary_emb=None, attention_mask=None):
        return torch.cat(_attend_stages((query, key, value), None, hidden_length, image_rotary_emb, attention_mask), dim=1)


def stage_ids(ref_dit, sample, encoder_attention_mask: torch.Tensor, hidden_length) -> list:
    """Per stage (seg, time) int32 [B, S_stage] of the reference's mask (F:320-350, M:348-378): seg 1 for valid tokens, 0 for
    padded text (encoder_attention_mask[i_p::num_stages]); time = the temporal order ids of the model's own
    _prepare_pyramid_image_ids (miniFLUX) or _prepare_pyramid_temporal_rope_ids (SD3 MMDiT), 0 for text, or 0 everywhere
    without use_temporal_causal."""
    num_stages = len(sample)
    first = sample[0][-1] if isinstance(sample[0], list) else sample[0]
    device, pad_bs = first.device, first.shape[0]
    order_ids = getattr(ref_dit, "_prepare_pyramid_temporal_rope_ids", None) or ref_dit._prepare_pyramid_image_ids
    image_ids = order_ids(sample, pad_bs, device) if ref_dit.use_temporal_causal else None
    out = []
    for i_p, length in enumerate(hidden_length):
        text = (encoder_attention_mask[i_p::num_stages] != 0).to(torch.int32)
        seg = torch.cat([text, torch.ones(pad_bs, length, dtype=torch.int32, device=text.device)], dim=1)
        time = torch.zeros_like(seg)
        if image_ids is not None:
            time[:, text.shape[1]:] = image_ids[i_p][:, :, 0].to(device=time.device, dtype=torch.int32)
        out.append((seg, time))
    return out


def _ref_module_attr(obj, name):
    return getattr(sys.modules[type(obj).__module__], name)


def install_training_attention(ref_dit) -> None:
    """Run every attention of an unmodified reference PyramidFluxTransformer or PyramidDiffusionMMDiT (use_flash_attn=False, no
    sequence parallelism, head_dim 64) on masked_attention.  Forward values are the reference's up to bf16 rounding inside the attention; the
    dense masks are no longer built into the saved graph.  Idempotent; undone by uninstall_training_attention."""
    if getattr(ref_dit, "_pf_training_attention", None) is not None:
        return
    if getattr(ref_dit, "use_flash_attn", False):
        raise ValueError("install_training_attention: the model runs the flash varlen path (use_flash_attn=True), which this "
                         "does not replace; build it with use_flash_attn=False, or use install_varlen_training_attention")
    if _ref_module_attr(ref_dit, "is_sequence_parallel_initialized")():
        raise ValueError("install_training_attention: sequence parallelism is initialised; its all-to-all attention path is "
                         "not replaced")
    head_dim = ref_dit.config.attention_head_dim
    if head_dim != HEAD_DIM:
        raise ValueError(f"install_training_attention: attention_head_dim {head_dim} unsupported ({HEAD_DIM} only)")

    saved = []
    for m in ref_dit.modules():
        proc = getattr(m, "processor", None)
        kind = type(proc).__name__
        if kind in ("FluxAttnProcessor2_0", "FluxSingleAttnProcessor2_0"):           # miniFLUX: the processors' callables
            saved.append((proc, "varlen_attn", proc.varlen_attn))
            proc.varlen_attn = _JointAttention() if kind == "FluxAttnProcessor2_0" else _SingleAttention()
        elif type(getattr(m, "var_len_attn", None)).__name__ == "VarlenSelfAttentionWithT5Mask":   # SD3 MMDiT: JointAttention's
            saved.append((m, "var_len_attn", m.var_len_attn))
            m.var_len_attn = _JointAttention()
    if not saved:
        raise TypeError(f"install_training_attention: no reference training attention found in {type(ref_dit).__name__}")

    had_own = "merge_input" in ref_dit.__dict__
    original = ref_dit.merge_input

    def merge_input(sample, encoder_hidden_length, encoder_attention_mask):
        res = list(original(sample, encoder_hidden_length, encoder_attention_mask))
        hidden_length = res[1]
        ids = stage_ids(ref_dit, sample, encoder_attention_mask, hidden_length)
        res[7] = [plan_for(seg, time) for seg, time in ids]      # the dense masks are dropped here
        return tuple(res)

    ref_dit.merge_input = merge_input
    ref_dit._pf_training_attention = (saved, had_own, original)


def uninstall_training_attention(ref_dit) -> None:
    """Restore what install_training_attention or install_varlen_training_attention changed on the instance."""
    state = getattr(ref_dit, "_pf_training_attention", None)
    if state is None:
        return
    saved, had_own, original = state
    for owner, name, fn in saved:
        setattr(owner, name, fn)
    if had_own:
        ref_dit.merge_input = original
    else:
        del ref_dit.merge_input
    del ref_dit._pf_training_attention


# ----------------------------------------------------------------------------------------------------------------------
# the flash varlen path: padding-free packed sequences, every stage in one attention launch
# ----------------------------------------------------------------------------------------------------------------------
class VarlenAttentionPlan:
    """The packed layout of one model call's attention, for every call site: `batch` sequences per stage of stage_len[i] rows
    (T + L_i) each; row_map int32 [total] (the padded position of each packed row, pf_b200.h pf_attn_varlen_layout) and pad_map
    int32 [batch * sum(stage_len)] (its inverse, -1 for dropped rows); the attention mask as seg / time int32 [1, total] (seg
    = sequence index + 1, stage-major then batch; time 0) with its tile schedules; cu_seqlens int32 [n_seq + 1] and
    max_seqlen as flash_attn takes them.  All tensors on one device."""

    def __init__(self, batch: int, stage_len, row_map, pad_map, seg, time, sched, kv_sched, cu_seqlens, max_seqlen: int):
        self.batch, self.stage_len = batch, list(stage_len)
        self.row_map, self.pad_map = row_map, pad_map
        self.seg, self.time, self.sched, self.kv_sched = seg, time, sched, kv_sched
        self.cu_seqlens, self.max_seqlen = cu_seqlens, max_seqlen

    @property
    def total(self) -> int:
        return self.row_map.numel()

    @property
    def shape(self) -> Tuple[int, int]:
        return tuple(self.seg.shape)


_VARLEN_PLANS: Dict[tuple, VarlenAttentionPlan] = {}


def varlen_plan(indices, seqlens, batch: int, stage_len, device=None) -> VarlenAttentionPlan:
    """The VarlenAttentionPlan of merge_input's flash branch (F:295-317): per stage i the `indices` into its flattened
    [batch, stage_len[i]] padding mask and `seqlens_in_batch` [batch].  Cached by content: one device-to-host copy per call."""
    n = len(stage_len)
    if not (len(indices) == len(seqlens) == n) or not 1 <= n <= _lib.VARLEN_MAX_STAGES:
        raise ValueError(f"varlen plan: {len(indices)} indices, {len(seqlens)} seqlens for {n} stages "
                         f"(1 .. {_lib.VARLEN_MAX_STAGES} stages)")
    device = torch.device(device) if device is not None else indices[0].device
    counts = [int(t.numel()) for t in indices]
    flat = torch.cat([t.detach().reshape(-1).to(torch.int64) for t in indices] +
                     [t.detach().reshape(-1).to(torch.int64) for t in seqlens]).cpu()       # the one device-to-host copy
    key = (str(device), batch, tuple(stage_len), tuple(counts), flat.numpy().tobytes())
    plan = _VARLEN_PLANS.get(key)
    if plan is not None:
        return plan
    idx, lens = flat[:sum(counts)], flat[sum(counts):].view(n, -1)
    if lens.shape[1] != batch:
        raise ValueError(f"varlen plan: seqlens_in_batch has {lens.shape[1]} entries per stage, the batch is {batch}")
    rows, off, pad0 = [], 0, 0
    for i, (c, length) in enumerate(zip(counts, stage_len)):
        ind = idx[off:off + c]
        # the rows of (stage i, batch b) are exactly seqlens[i][b] increasing indices inside b's padded sequence
        if c and (bool((ind[1:] <= ind[:-1]).any()) or int(ind[0]) < 0 or int(ind[-1]) >= batch * length
                  or not torch.equal(torch.bincount(ind // length, minlength=batch), lens[i])):
            raise ValueError(f"varlen plan: stage {i}'s indices do not match its seqlens_in_batch {lens[i].tolist()}")
        rows.append(ind + pad0)
        off, pad0 = off + c, pad0 + batch * length
    if not bool((lens > 0).all()):
        raise ValueError("varlen plan: every sequence needs at least one row")
    plan = _make_varlen_plan(batch, stage_len, torch.cat(rows), lens.reshape(-1), device)
    if len(_VARLEN_PLANS) >= _PLAN_CACHE_SIZE:
        _VARLEN_PLANS.clear()
    _VARLEN_PLANS[key] = plan
    return plan


def _make_varlen_plan(batch: int, stage_len, row_map: torch.Tensor, seqlens: torch.Tensor, device) -> VarlenAttentionPlan:
    """The plan of a (CPU) row map whose packed rows hold sequences of the given lengths, one after the other."""
    total = row_map.numel()
    pad_map = torch.full((batch * sum(stage_len),), -1, dtype=torch.int32)
    pad_map[row_map.long()] = torch.arange(total, dtype=torch.int32)
    seg = torch.repeat_interleave(torch.arange(1, seqlens.numel() + 1, dtype=torch.int32), seqlens)[None]
    time = torch.zeros_like(seg)
    sched, _ = ops.attn_build_schedule(seg, time)
    kv_sched = ops.attn_build_kv_schedule(sched, total)
    cu = torch.nn.functional.pad(torch.cumsum(seqlens, 0), (1, 0)).to(torch.int32)
    return VarlenAttentionPlan(batch, stage_len, row_map.to(device, torch.int32), pad_map.to(device), seg.to(device),
                               time.to(device), sched.to(device), kv_sched.to(device), cu.to(device), int(seqlens.max()))


class _VarlenPack(torch.autograd.Function):
    """Every stage of one call site packed into head-major q / k / v [1, H, total, 64] (pf_attn_varlen_pack); the backward
    (pf_attn_varlen_pack_bwd) writes every row of every source gradient once, 0 for the dropped rows."""

    @staticmethod
    def forward(ctx, plan: VarlenAttentionPlan, stage_row0, has_text: bool, *tensors):
        video = tensors[:3]
        text = tensors[3:6] if has_text else None
        freqs = tensors[6 if has_text else 3:] or None
        h = video[0].shape[2]
        packed = tuple(torch.empty(1, h, plan.total, HEAD_DIM, dtype=torch.bfloat16, device=video[0].device) for _ in range(3))
        ops.attn_varlen_pack(video, text, freqs, packed, stage_len=plan.stage_len, stage_row0=stage_row0,
                             row_map=plan.row_map, pad_map=plan.pad_map)
        ctx.plan, ctx.stage_row0, ctx.has_text = plan, stage_row0, has_text
        ctx.sources = [(t.shape, t.dtype) for t in tensors[:6 if has_text else 3]]
        if freqs is not None:
            ctx.save_for_backward(*freqs)
        return packed

    @staticmethod
    def backward(ctx, *grads):
        freqs = ctx.saved_tensors or None
        dev = grads[0].device
        dsrc = [torch.empty(shape, dtype=dt, device=dev) for shape, dt in ctx.sources]
        plan = ctx.plan
        ops.attn_varlen_pack(tuple(dsrc[:3]), tuple(dsrc[3:]) if ctx.has_text else None, freqs,
                             tuple(g.contiguous() for g in grads), stage_len=plan.stage_len, stage_row0=ctx.stage_row0,
                             row_map=plan.row_map, pad_map=plan.pad_map, bwd=True)
        return (None, None, None, *dsrc) + (None,) * (0 if freqs is None else len(freqs))


class _VarlenUnpack(torch.autograd.Function):
    """The packed attention output [1, total, H*64] scattered into the call site's outputs (pf_attn_varlen_unpack, zeros for
    dropped rows); the backward gathers the output gradients into the packed dout (pf_attn_varlen_unpack_bwd)."""

    @staticmethod
    def forward(ctx, plan: VarlenAttentionPlan, stage_row0, out, video_shape, video_dtype, text_shape, text_dtype):
        video = torch.empty(video_shape, dtype=video_dtype, device=out.device)
        text = torch.empty(text_shape, dtype=text_dtype, device=out.device) if text_shape is not None else None
        ops.attn_varlen_unpack(video, text, out, stage_len=plan.stage_len, stage_row0=stage_row0, row_map=plan.row_map,
                               pad_map=plan.pad_map)
        ctx.plan, ctx.stage_row0 = plan, stage_row0
        return (video, text) if text is not None else video

    @staticmethod
    def backward(ctx, dvideo, dtext=None):
        plan = ctx.plan
        grads = [g if ops.attn_varlen_rows_ok(g) else g.contiguous() for g in ((dvideo, dtext) if dtext is not None else (dvideo,))]
        dout = torch.empty(1, plan.total, grads[0].shape[-1], dtype=torch.bfloat16, device=grads[0].device)
        ops.attn_varlen_unpack(grads[0], grads[1] if len(grads) > 1 else None, dout, stage_len=plan.stage_len,
                               stage_row0=ctx.stage_row0, row_map=plan.row_map, pad_map=plan.pad_map, bwd=True)
        return None, None, dout, None, None, None, None


def _check_varlen_sources(sources) -> None:
    for t in sources:
        if t.ndim != 4 or t.shape[-1] != HEAD_DIM:
            raise ValueError(f"varlen attention: q / k / v must be [B, S, H, {HEAD_DIM}] (got {tuple(t.shape)})")
        if t.dtype not in (torch.bfloat16, torch.float32):
            raise ValueError(f"varlen attention: q / k / v must be bf16 or fp32 (got {t.dtype})")
    if not sources[0].is_cuda:
        raise RuntimeError("varlen attention runs on the GPU only (pyramid_flow_b200 has no CPU path)")
    _lib.require_device()


def _attend_varlen(plan: VarlenAttentionPlan, video, text, stage_row0, image_rotary_emb, scale: float, out_dtypes):
    sources = tuple(video) + (tuple(text) if text is not None else ())
    sources = tuple(t if ops.attn_pack_source_ok(t) else t.contiguous() for t in sources)
    freqs = tuple(image_rotary_emb[i] for i in range(len(plan.stage_len))) if image_rotary_emb is not None else ()
    q, k, v = _VarlenPack.apply(plan, stage_row0, text is not None, *sources, *freqs)
    out = _MaskedAttention.apply(q, k, v, plan, float(scale))
    b, s, h, hd = video[0].shape
    text_shape = None if text is None else (text[0].shape[0], text[0].shape[1], h * hd)
    return _VarlenUnpack.apply(plan, stage_row0, out, (b, s, h * hd), out_dtypes[0], text_shape, out_dtypes[1])


def _varlen_plan_arg(encoder_attention_mask) -> VarlenAttentionPlan:
    if not isinstance(encoder_attention_mask, VarlenAttentionPlan):
        raise TypeError("the installed varlen training attention takes the VarlenAttentionPlan of the wrapped merge_input, got "
                        f"{type(encoder_attention_mask).__name__} (was the model's merge_input replaced after "
                        "install_varlen_training_attention?)")
    return encoder_attention_mask


def _check_stages(plan: VarlenAttentionPlan, video, text_len: int, seq_lens) -> None:
    if [text_len + n for n in seq_lens] != plan.stage_len or video[0].shape[0] != plan.batch or \
            sum(seq_lens) != video[0].shape[1]:
        raise ValueError(f"varlen attention: the plan is for batch {plan.batch}, stages {plan.stage_len}; the call site has "
                         f"{tuple(video[0].shape)} with text {text_len}, stages {list(seq_lens)}")


class _VarlenJointAttention:
    """Stands for VarlenFlashSelfAttentionWithT5Mask (B:189-263): per stage i_p its text rows (encoder rows i_p::stages) then
    its video rows, apply_rope with image_rotary_emb[i_p], the padded text rows dropped; one attention over every (stage,
    batch) sequence; outputs scattered back, zeros for dropped rows."""

    def __call__(self, query, key, value, encoder_query, encoder_key, encoder_value, heads, scale, hidden_length=None,
                 image_rotary_emb=None, encoder_attention_mask=None):
        plan = _varlen_plan_arg(encoder_attention_mask)
        video, text = (query, key, value), (encoder_query, encoder_key, encoder_value)
        _check_varlen_sources(video + text)
        text_len = encoder_query.shape[1]
        _check_stages(plan, video, text_len, hidden_length)
        if encoder_query.shape[0] != plan.batch * len(hidden_length):
            raise ValueError(f"varlen attention: text q / k / v {tuple(encoder_query.shape)} for batch {plan.batch} and "
                             f"{len(hidden_length)} stages")
        stage_row0 = [sum(hidden_length[:i]) for i in range(len(hidden_length))]
        return _attend_varlen(plan, video, text, stage_row0, image_rotary_emb, scale, (query.dtype, encoder_query.dtype))


class _VarlenSingleAttention:
    """Stands for VarlenFlashSelfAttnSingle (B:452-516): the single blocks' joint sequence is already stage-major."""

    def __call__(self, query, key, value, heads, scale, hidden_length=None, image_rotary_emb=None, encoder_attention_mask=None):
        plan = _varlen_plan_arg(encoder_attention_mask)
        video = (query, key, value)
        _check_varlen_sources(video)
        _check_stages(plan, video, 0, hidden_length)
        stage_row0 = [sum(hidden_length[:i]) for i in range(len(hidden_length))]
        return _attend_varlen(plan, video, None, stage_row0, image_rotary_emb, scale, (query.dtype, None))


_IDENTITY_PLANS: Dict[tuple, VarlenAttentionPlan] = {}


def varlen_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens: torch.Tensor,
                     softmax_scale: Optional[float] = None) -> torch.Tensor:
    """The subset of flash_attn_varlen_func the reference calls: non-causal self-attention within each sequence
    [cu_seqlens[j], cu_seqlens[j + 1]), equal q and k lengths, no dropout, head_dim 64.  q, k, v token-major [total, H, 64]
    (bf16 or fp32, rounded once to bf16); returns [total, H, 64] in q's dtype, differentiable w.r.t. q, k, v.
    softmax_scale defaults to 64 ** -0.5."""
    sources = tuple(t.unsqueeze(0) for t in (q, k, v))
    if not (q.shape == k.shape == v.shape) or q.ndim != 3:
        raise ValueError(f"varlen_attention: q, k, v must all be [total, H, {HEAD_DIM}] (got {q.shape}, {k.shape}, {v.shape})")
    _check_varlen_sources(sources)
    total = q.shape[0]
    cu = cu_seqlens.detach().to("cpu", torch.int64)
    if cu.ndim != 1 or cu.numel() < 2 or int(cu[0]) != 0 or int(cu[-1]) != total or bool((cu[1:] <= cu[:-1]).any()):
        raise ValueError(f"varlen_attention: cu_seqlens must rise strictly from 0 to total = {total} (got {cu.tolist()})")
    key = (str(q.device), cu.numpy().tobytes())
    plan = _IDENTITY_PLANS.get(key)
    if plan is None:        # one stage of one batch row holding every sequence: the identity row map
        plan = _make_varlen_plan(1, [total], torch.arange(total), cu[1:] - cu[:-1], q.device)
        if len(_IDENTITY_PLANS) >= _PLAN_CACHE_SIZE:
            _IDENTITY_PLANS.clear()
        _IDENTITY_PLANS[key] = plan
    scale = HEAD_DIM ** -0.5 if softmax_scale is None else softmax_scale
    out = _attend_varlen(plan, sources, None, [0], None, scale, (q.dtype, None))
    return out.view(total, q.shape[1], HEAD_DIM)


def install_varlen_training_attention(ref_dit) -> None:
    """Run every attention of an unmodified reference PyramidFluxTransformer built with use_flash_attn=True (no sequence
    parallelism, head_dim 64) on the library: the processors' varlen_flash_attn callables are replaced, merge_input's entry 6
    (the per-stage indices / seqlens_in_batch dicts) becomes one VarlenAttentionPlan.  Forward values are the reference's up
    to bf16 rounding inside the attention; flash_attn is not needed.  Idempotent; undone by uninstall_training_attention."""
    if getattr(ref_dit, "_pf_training_attention", None) is not None:
        return
    if type(ref_dit).__name__ != "PyramidFluxTransformer":
        raise ValueError(f"install_varlen_training_attention: {type(ref_dit).__name__} is not a miniFLUX PyramidFluxTransformer "
                         "(the SD3 MMDiT cannot train on its flash path: it refuses use_flash_attn with use_temporal_causal)")
    if not getattr(ref_dit, "use_flash_attn", False):
        raise ValueError("install_varlen_training_attention: the model runs the SDPA path (use_flash_attn=False); use "
                         "install_training_attention")
    if _ref_module_attr(ref_dit, "is_sequence_parallel_initialized")():
        raise ValueError("install_varlen_training_attention: sequence parallelism is initialised; its all-to-all flash path "
                         "is not replaced")
    head_dim = ref_dit.config.attention_head_dim
    if head_dim != HEAD_DIM:
        raise ValueError(f"install_varlen_training_attention: attention_head_dim {head_dim} unsupported ({HEAD_DIM} only)")

    saved = []
    for m in ref_dit.modules():
        proc = getattr(m, "processor", None)
        kind = type(proc).__name__
        if kind in ("FluxAttnProcessor2_0", "FluxSingleAttnProcessor2_0"):
            saved.append((proc, "varlen_flash_attn", proc.varlen_flash_attn))
            proc.varlen_flash_attn = _VarlenJointAttention() if kind == "FluxAttnProcessor2_0" else _VarlenSingleAttention()
    if not saved:
        raise TypeError(f"install_varlen_training_attention: no flash attention processor found in {type(ref_dit).__name__}")

    had_own = "merge_input" in ref_dit.__dict__
    original = ref_dit.merge_input

    def merge_input(sample, encoder_hidden_length, encoder_attention_mask):
        res = list(original(sample, encoder_hidden_length, encoder_attention_mask))
        stages = res[6]
        text_len = encoder_attention_mask.shape[1]
        res[6] = varlen_plan([st["indices"] for st in stages], [st["seqlens_in_batch"] for st in stages],
                             int(stages[0]["seqlens_in_batch"].numel()), [text_len + n for n in res[1]])
        return tuple(res)

    ref_dit.merge_input = merge_input
    ref_dit._pf_training_attention = (saved, had_own, original)
