"""Identity-V probes of the masked attention kernels (pf_attn_fwd_masked, pf_attn_bwd_masked, pf_attn_fwd_text).

With H = ceil(S / 64) heads, head h "owns" keys [64 h, 64 h + 64).  Give every head the one-hot value rows
v[b, h, kv, :] = e_(kv - 64 h) on the keys it owns and zeros elsewhere; then for any q and k

    out[b, q, 64 h + d] = P_{b,h}[q, 64 h + d]        and        out[b, q, j] = 0 for j >= S,

so one launch prints the whole S x S probability matrix, column kv taken from head kv // 64.  The same trick on the other
operands prints the backward's matrices: an identity dO gives dV = P^T, an identity K gives dQ = scale dS, an identity Q
gives dK = scale dS^T.  Every element is then compared with an fp64 attention of the same bf16 inputs:

    masked pair   -> exactly 0 (a skipped tile and a masked column both give an exact 0 in the kernels)
    allowed pair  -> P: strictly > 0 and within a relative bound;  dS: within an absolute bound, and non-zero with the
                     reference's sign wherever |dS| clears that bound.

Everything here runs on the CPU as well as on the GPU (tests/test_attn_probe_cpu.py checks the harness itself)."""
from __future__ import annotations

from dataclasses import dataclass

import torch

SCALE = 0.125
SENTINEL = 7.0          # exactly representable in bf16; marks output the kernel must leave alone

# ---- error bounds ------------------------------------------------------------------------------------------------------
# The kernels' arithmetic, per probed element (u_bf16 = 2^-8, the unit roundoff of bf16's 8-bit significand):
#   scores   fp32 wgmma accumulation of 64 exact bf16 products: |error| <= EPS_ACC * sum_i |q_i k_i| <= EPS_ACC |q| |k|
#            (EPS_ACC = 2^-17 is twice the classic 64 * 2^-24 bound, room for a truncating accumulator).  p = exp(scale s - m)
#            carries the score error of its own column and of the row's max (or lse): relative 2 scale EPS_ACC |q| |k|.
#   fp32     ex2.approx (2^-22), rounding of the exp2 arguments and of lse (magnitudes < 32), the row sum l (chains of a
#            few hundred fp32 additions): together below ETA_FP32 = 2^-14 relative.
#   forward  out = bf16(bf16(p) * (1 / l)): two bf16 roundings, (1 + 2^-8)^2 - 1 = 2^-7 + 2^-16 relative.
#   dV       bf16(p) times a one-hot dO row: one bf16 rounding, 2^-8 relative.
#   dQ, dK   bf16(p (dP - delta)) times a one-hot K / Q row and a power-of-two scale: one bf16 rounding of dS, plus the fp32
#            accumulation errors of dP = dO.v (<= EPS_ACC |dO| |v|) and delta = dO.O (<= EPS_ACC |dO| |O|) times p.
EPS_ACC = 2.0 ** -17
ETA_FP32 = 2.0 ** -14


def eta_p(scale: float, qk_norm_max: float) -> float:
    """Relative error of a kernel's fp32 probability before any bf16 rounding."""
    return 2.0 * scale * EPS_ACC * qk_norm_max + ETA_FP32


def rel_bound_fwd(scale: float, qk_norm_max: float) -> float:
    """Relative bound of a probed forward probability out = bf16(bf16(p) / l) against fp64."""
    return 2.0 ** -7 + 2.0 ** -16 + eta_p(scale, qk_norm_max)


def rel_bound_dv(scale: float, qk_norm_max: float) -> float:
    """Relative bound of a probed dV = bf16(p) against fp64."""
    return 2.0 ** -8 + eta_p(scale, qk_norm_max)


def norm_product_max(q: torch.Tensor, k: torch.Tensor) -> float:
    """max over pairs of |q_row| |k_row| (>= sum_i |q_i k_i| by Cauchy-Schwarz), over all heads."""
    return (q.double().norm(dim=-1).amax() * k.double().norm(dim=-1).amax()).item()


# ---- probe tensors -----------------------------------------------------------------------------------------------------
def heads_for(seq: int) -> int:
    return (seq + 63) // 64


def identity_heads(batch: int, seq: int, heads: int, device) -> torch.Tensor:
    """bf16 [batch, heads, seq, 64]: row r of head h is e_(r - 64 h) on the rows head h owns, zero elsewhere."""
    eye = torch.eye(seq, heads * 64, dtype=torch.bfloat16, device=device)
    return eye.view(seq, heads, 64).transpose(0, 1).unsqueeze(0).expand(batch, -1, -1, -1).contiguous()


def random_heads(batch: int, seq: int, heads: int, gen: torch.Generator, device, distinct: bool = True) -> torch.Tensor:
    """bf16 [batch, heads, seq, 64] ~ N(0, 1); distinct=False copies one head to all (the fp64 reference is then one matrix)."""
    x = torch.randn(batch, heads if distinct else 1, seq, 64, generator=gen)
    return x.to(device, torch.bfloat16).expand(-1, heads, -1, -1).contiguous()


def head_columns(x: torch.Tensor) -> torch.Tensor:
    """[B, H, S, 64] -> [B, S, H * 64]: column 64 h + d is dim d of head h (the layout of the forward's output)."""
    b, h, s, d = x.shape
    return x.transpose(1, 2).reshape(b, s, h * d)


def dense_mask(seg: torch.Tensor, time: torch.Tensor) -> torch.Tensor:
    """Allowed pairs [B, S, S] = same segment and time_kv <= time_q (the attention's mask definition)."""
    return (seg[:, :, None] == seg[:, None, :]) & (time[:, :, None] >= time[:, None, :])


# ---- fp64 references ---------------------------------------------------------------------------------------------------
def _probs(q: torch.Tensor, k: torch.Tensor, allowed: torch.Tensor, scale: float, h: int, bias=None):
    s = (q[:, h].double() @ k[:, h].double().transpose(-1, -2)) * scale
    if bias is not None:                # T5's relative position bias as a Toeplitz table [heads, 2 S - 1]: kv - q + S - 1
        n = s.shape[-1]
        idx = torch.arange(n, device=s.device)[None, :] - torch.arange(n, device=s.device)[:, None] + n - 1
        s = s + bias[h].double()[idx]
    s = s.masked_fill(~allowed, float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    return torch.exp(s - lse[..., None]), lse


def fwd_reference(q: torch.Tensor, k: torch.Tensor, allowed: torch.Tensor, scale: float, distinct: bool = True, bias=None):
    """-> (P fp64 [B, S, S] with column kv taken from head kv // 64, lse fp64 [B, H, S]).  bias: optional fp32 [H, 2 S - 1]."""
    b, heads, s, _ = q.shape
    if not distinct:
        assert bias is None
        p, lse = _probs(q, k, allowed, scale, 0)
        return p, lse[:, None].expand(b, heads, s)
    p = torch.zeros(b, s, s, dtype=torch.float64, device=q.device)
    lses = []
    for h in range(heads):
        ph, lh = _probs(q, k, allowed, scale, h, bias)
        lses.append(lh)
        if 64 * h < s:
            c = slice(64 * h, min(s, 64 * h + 64))
            p[:, :, c] = ph[:, :, c]
    return p, torch.stack(lses, 1)


@dataclass
class BwdReference:
    """fp64 composites of the three backward probes, each [B, S, S]: column j taken from head j // 64.
    pt[b, kv, q] = P_{q//64}[q, kv] (dV probe), ds[b, q, kv] = dS_{kv//64}[q, kv] (dQ probe),
    dst[b, kv, q] = dS_{q//64}[q, kv] (dK probe); ds_bound / dst_bound: the elementwise error bounds of the kernel's dS."""
    pt: torch.Tensor
    ds: torch.Tensor
    ds_bound: torch.Tensor
    dst: torch.Tensor
    dst_bound: torch.Tensor
    rel_dv: float


def bwd_reference(q, k, v, out, dout, allowed, scale: float) -> BwdReference:
    """q, k, v bf16 [B, H, S, 64]; out / dout bf16 [B, S, H * 64] (out: what the forward wrote: delta is taken from it, as the
    kernel's contract states)."""
    b, heads, s, _ = q.shape
    o = out.double().view(b, s, heads, 64).transpose(1, 2)
    do = dout.double().view(b, s, heads, 64).transpose(1, 2)
    eta = eta_p(scale, norm_product_max(q, k))
    z = lambda: torch.zeros(b, s, s, dtype=torch.float64, device=q.device)
    ref = BwdReference(z(), z(), z(), z(), z(), 2.0 ** -8 + eta)
    for h in range(heads):
        p, _ = _probs(q, k, allowed, scale, h)
        vh = v[:, h].double()
        delta = (do[:, h] * o[:, h]).sum(-1)
        ds = p * (do[:, h] @ vh.transpose(-1, -2) - delta[..., None])
        acc = do[:, h].norm(dim=-1)[:, :, None] * (vh.norm(dim=-1)[:, None, :] + o[:, h].norm(dim=-1)[:, :, None])
        bound = (2.0 ** -8 + eta + 2.0 ** -22) * ds.abs() + (1 + 2.0 ** -7) * p * EPS_ACC * acc
        if 64 * h >= s:
            continue
        c = slice(64 * h, min(s, 64 * h + 64))
        ref.pt[:, :, c] = p[:, c, :].transpose(1, 2)
        ref.ds[:, :, c] = ds[:, :, c]
        ref.ds_bound[:, :, c] = bound[:, :, c]
        ref.dst[:, :, c] = ds[:, c, :].transpose(1, 2)
        ref.dst_bound[:, :, c] = bound[:, c, :].transpose(1, 2)
    return ref


# ---- checks ------------------------------------------------------------------------------------------------------------
@dataclass
class Report:
    """Violations of one probe, as bool maps [B, S, W] over (batch, row, column):
    leaked  - a masked pair (or a column past the sequence) holds a non-zero value;
    missing - an allowed pair that must be non-zero is zero (P), or is zero / has the wrong sign where |ref| clears the
              bound (dS);
    inexact - an allowed pair outside the error bound.
    worst: the worst relative error against fp64 over the allowed pairs (dS: over those with |ref| >= max |ref| / 16);
    rel_bound: the relative bound asserted (P); bound_use: the largest error as a fraction of its elementwise bound (dS)."""
    name: str
    leaked: torch.Tensor
    missing: torch.Tensor
    inexact: torch.Tensor
    worst: float
    rel_bound: float | None = None
    bound_use: float | None = None

    def exact_violations(self) -> torch.Tensor:
        return self.leaked | self.missing

    def any(self) -> torch.Tensor:
        return self.leaked | self.missing | self.inexact

    def ok(self) -> bool:
        return not bool(self.any().any())

    def __str__(self) -> str:
        lim = (f"bound {self.rel_bound:.3e}" if self.rel_bound is not None else f"{self.bound_use:.2f} of the error bound used")
        lines = [f"{self.name}: worst relative error {self.worst:.3e} ({lim})"]
        for kind in ("leaked", "missing", "inexact"):
            m = getattr(self, kind)
            n = int(m.sum())
            if n == 0:
                continue
            idx = m.nonzero()
            lo, hi = idx.amin(0).tolist(), idx.amax(0).tolist()
            first = ", ".join(str(tuple(i)) for i in idx[:4].tolist())
            lines.append(f"  {kind}: {n} elements (batch, row, col) in batches {lo[0]}..{hi[0]}, rows {lo[1]}..{hi[1]}, "
                         f"cols {lo[2]}..{hi[2]}; first {first}")
        return "\n".join(lines)


def pad_cols(x: torch.Tensor, width: int, value) -> torch.Tensor:
    if x.shape[-1] == width:
        return x
    pad = torch.full((*x.shape[:-1], width - x.shape[-1]), value, dtype=x.dtype, device=x.device)
    return torch.cat([x, pad], -1)


def check_probs(name: str, got: torch.Tensor, ref: torch.Tensor, allowed: torch.Tensor, rel_bound: float) -> Report:
    """got [B, S, W >= S] (columns >= S must be exactly 0), ref fp64 [B, S, S], allowed bool [B, S, S]."""
    width = got.shape[-1]
    ref = pad_cols(ref, width, 0.0)
    allowed = pad_cols(allowed, width, False)
    g = got.double()
    err = (g - ref).abs()
    rel = torch.where(allowed, err / ref.clamp_min(1e-300), torch.zeros_like(err))
    return Report(name, ~allowed & (g != 0), allowed & ~(g > 0), allowed & (err > rel_bound * ref),
                  rel.max().item() if rel.numel() else 0.0, rel_bound=rel_bound)


def check_grads(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, allowed: torch.Tensor) -> Report:
    """got [B, S, W >= S] (columns >= S must be exactly 0), ref / bound fp64 [B, S, S], allowed bool [B, S, S]."""
    width = got.shape[-1]
    ref = pad_cols(ref, width, 0.0)
    bound = pad_cols(bound, width, 0.0)
    allowed = pad_cols(allowed, width, False)
    g = got.double()
    err = (g - ref).abs()
    clear = allowed & (ref.abs() > bound)
    big = allowed & (ref.abs() >= ref.abs().amax() / 16)
    rel = torch.where(big, err / ref.abs().clamp_min(1e-300), torch.zeros_like(err))
    use = torch.where(allowed, err / bound.clamp_min(1e-300), torch.zeros_like(err))
    return Report(name, ~allowed & (g != 0), clear & ~(g * ref.sign() > 0), allowed & (err > bound),
                  rel.max().item() if rel.numel() else 0.0, bound_use=use.max().item() if use.numel() else 0.0)


# ---- layouts -----------------------------------------------------------------------------------------------------------
def restated_layout(batch: int, text: int, clips, causal: bool = True):
    """seg / time [batch, S] int32 of the training tests' layouts: text padded differently per sample (sample b keeps
    text - 7 (b + 1) valid tokens when text > 16), then clips (frames, tokens per frame) with one time stamp per frame."""
    segs, times = [], []
    for b in range(batch):
        valid = text - 7 * (b + 1) if text > 16 else text
        seg = [1] * valid + [0] * (text - valid)
        time = [0] * text
        stamp = 0
        for t, n in clips:
            for f in range(t):
                seg += [1] * n
                time += [(stamp + f) if causal else 0] * n
            stamp += t
        segs.append(seg)
        times.append(time)
    return torch.tensor(segs, dtype=torch.int32), torch.tensor(times, dtype=torch.int32)


def random_ids_layout(batch: int, seq: int, gen: torch.Generator):
    """seg in {0, 1, 2}, time in {0..3}, drawn per token: every tile partial, masks with holes."""
    return (torch.randint(0, 3, (batch, seq), generator=gen, dtype=torch.int32),
            torch.randint(0, 4, (batch, seq), generator=gen, dtype=torch.int32))


# ---- schedule mutations (for the sensitivity tests) --------------------------------------------------------------------
def sched_entries(sched: torch.Tensor) -> set:
    """{(batch, row tile, column tile, partial flag)} of a tile schedule [B, tiles, stride] (q-major or kv-major)."""
    out = set()
    for b in range(sched.shape[0]):
        for t in range(sched.shape[1]):
            row = sched[b, t]
            for e in row[1:1 + int(row[0])].tolist():
                out.add((b, t, e >> 1, e & 1))
    return out


def drop_entry(sched: torch.Tensor, b: int, t: int, i: int) -> torch.Tensor:
    """A copy of the schedule with entry i of row (b, t) removed (the row stays packed and zero-padded)."""
    s = sched.clone()
    n = int(s[b, t, 0])
    assert 0 <= i < n
    s[b, t, 1 + i:n] = sched[b, t, 2 + i:n + 1].clone()
    s[b, t, n] = 0
    s[b, t, 0] = n - 1
    return s


def clear_partial(sched: torch.Tensor, b: int, t: int, i: int) -> torch.Tensor:
    """A copy of the schedule with the partial flag of entry i of row (b, t) cleared (the tile is then treated as full)."""
    s = sched.clone()
    assert 0 <= i < int(s[b, t, 0]) and int(s[b, t, 1 + i]) & 1
    s[b, t, 1 + i] = int(s[b, t, 1 + i]) & ~1
    return s


def tile_region(shape, b: int, rows: int, cols: int | None = None, tile: int = 128) -> torch.Tensor:
    """bool [B, S, W]: True on row tile `rows` of batch b (and column tile `cols`, if given)."""
    m = torch.zeros(shape, dtype=torch.bool)
    c = slice(None) if cols is None else slice(cols * tile, (cols + 1) * tile)
    m[b, rows * tile:(rows + 1) * tile, c] = True
    return m
