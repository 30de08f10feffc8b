// pf_attn.cu — masked joint text+video attention forward on Hopper warpgroup MMA (head_dim 64).
//
//   out[b, q, h, :] = softmax_kv( q.k * scale  | mask(q, kv) ) . v ,   mask = (seg_q == seg_kv) && (time_q >= time_kv)
//
// replaces F.scaled_dot_product_attention with the dense [B,1,S,S] bool mask (reference B:363-365, B:596-598; mask
// built at F:318-350).  The mask is never materialised: a host-built tile schedule (pf_attn_build_schedule) lists, per
// 128-row q tile, only the 128-wide kv tiles that contain an allowed pair and flags the few that need an element mask.
//
// One CTA = one (batch, head, 128-row q tile); 384 threads:
//   warpgroup 0 (one lane)  TMA producer: Q once, then K and V tiles through 2-stage mbarrier rings
//   warpgroups 1, 2         64 q rows each: S = Q.K^T (wgmma, both operands in smem, K-major) lands in registers, the online
//                           softmax (exact running max, exp2) runs on the accumulator fragments, P is re-packed in registers as
//                           the bf16 A operand and O += P.V is a wgmma with A from registers and V from smem MN-major -- V is
//                           consumed in its natural [kv, hd] layout, no transpose.
//
// Schedule of a consumer warpgroup, iteration j (tile 0 issues S(0) alone, and the last P.V is issued after the loop):
//   wait K(j), V(j-1); [turn] issue S(j) = Q.K(j)^T and O += P(j-1).V(j-1) as two wgmma groups; [hand the turn over]
//   wait for S(j) only, release K(j); mask + softmax of tile j (the exponentials run under P(j-1).V(j-1));
//   wait for P(j-1).V(j-1), release V(j-1); O *= alpha(j); pack P(j).
// The two warpgroups take turns at the tensor core (named barriers 1 and 2), so one warpgroup's softmax also runs under
// the other's MMAs.
// Two stages suffice and cannot deadlock: the producer loads K(0), V(0), K(1), V(1), ...; iteration j needs K(j) and
// V(j-1), and loading them needs only the releases of K(j-2) and V(j-3), made in iteration j-2 by both warpgroups.  A
// warpgroup waiting in iteration j has taken its turn j-1, so the other one has taken at least its turn j-2 and can finish
// iteration j-2 without waiting for anything more.
#include <algorithm>
#include <vector>

#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

constexpr int ATT_BM = 128;      // q rows per CTA
constexpr int ATT_BN = 128;      // kv columns per tile
constexpr int ATT_HD = 64;
constexpr int ATT_STAGES = 2;
constexpr int ATT_THREADS = 384;
constexpr int ATT_TILE_BYTES = ATT_BN * ATT_HD * 2;  // 16 KB
constexpr int ATT_SMEM_BYTES = (1 + 2 * ATT_STAGES) * ATT_TILE_BYTES + 1024;

struct AttnArgs {
  __nv_bfloat16* out;
  long long ldo;
  int batch, heads, seq, q_tiles;
  float scale_log2;
  const int* seg;
  const int* time;
  const int* sched;
  int sched_stride;
  // sequence parallel: output rows go straight into the owning rank's buffer (pf_b200.h)
  __nv_bfloat16* peer_out[PF_MAX_PEERS];
  int peer_count, peer_chunk_rows, peer_col_begin;
  // fp32 [batch, heads, seq]: natural-log log-sum-exp of each row's scaled scores (the attention backward's softmax statistic)
  float* lse;
};

// kLse: also store each row's log-sum-exp.  A template flag, so the launches without it run exactly the code they always ran.
template <bool kLse>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                const __grid_constant__ CUtensorMap tm_v, const AttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_k = smem + ATT_TILE_BYTES;
  uint8_t* smem_v = smem_k + ATT_STAGES * ATT_TILE_BYTES;

  __shared__ __align__(8) uint64_t bar_q;
  __shared__ __align__(8) uint64_t k_full[ATT_STAGES], k_empty[ATT_STAGES], v_full[ATT_STAGES], v_empty[ATT_STAGES];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wgroup = warp >> 2;
  // heavy (late) q tiles first: they own the longest kv lists
  const int qt = a.q_tiles - 1 - static_cast<int>(blockIdx.x);
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int bh = b * a.heads + h;
  const int* sched = a.sched + (static_cast<size_t>(b) * a.q_tiles + qt) * a.sched_stride;
  const int n_kv = sched[0];

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    mbar_init(&bar_q, 1);
    for (int i = 0; i < ATT_STAGES; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);   // one arrival per consumer warp
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wgroup == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // ===== TMA producer =====
      mbar_arrive_expect_tx(&bar_q, ATT_TILE_BYTES);
      tma_load_3d(smem_q, &tm_q, &bar_q, 0, qt * ATT_BM, bh);
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < n_kv; ++j) {
        const int kt = sched[1 + j] >> 1;
        mbar_wait(&k_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&k_full[st], ATT_TILE_BYTES);
        tma_load_3d(smem_k + st * ATT_TILE_BYTES, &tm_k, &k_full[st], 0, kt * ATT_BN, bh);
        mbar_wait(&v_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&v_full[st], ATT_TILE_BYTES);
        tma_load_3d(smem_v + st * ATT_TILE_BYTES, &tm_v, &v_full[st], 0, kt * ATT_BN, bh);
        if (++st == ATT_STAGES) {
          st = 0;
          ph ^= 1;
        }
      }
    }
    return;
  }

  // ===== consumers: thread (warp w of the warpgroup, g = lane / 4, t = lane % 4) holds rows r0 = 16 w + g and r0 + 8 of its
  // warpgroup's 64 q rows, columns 8 i + 2 t, 8 i + 2 t + 1 of every 8-column group i (the wgmma accumulator fragment) =====
  setmaxnreg_inc<232>();
  const int wg = wgroup - 1;
  const int g4 = lane >> 2, t4 = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + g4;
  const float c = a.scale_log2;
  const int* sg = a.seg + static_cast<size_t>(b) * a.seq;
  const int* tm = a.time + static_cast<size_t>(b) * a.seq;
  int seg_q[2], time_q[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qpos = qt * ATT_BM + row0 + 8 * r;
    const bool q_valid = qpos < a.seq;
    seg_q[r] = q_valid ? sg[qpos] : -0x7fffffff;
    time_q[r] = q_valid ? tm[qpos] : -0x7fffffff;
  }
  float m_run[2] = {-INFINITY, -INFINITY};   // running row max (raw score units); -inf: no allowed score seen yet
  float l_run[2] = {0.f, 0.f};               // this thread's part of the row sum (its 32 of every tile's 128 columns)
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;

  mbar_wait(&bar_q, 0);
  const uint64_t dq = make_smem_desc_kmajor_sw128(smem_u32(smem_q) + wg * (64 * 128));

  // S = Q.K^T of the tile in `stage`: one wgmma group.  The caller fences.
  auto issue_qk = [&](float (&s)[64], int stage) {
    const uint64_t dk = make_smem_desc_kmajor_sw128(smem_u32(smem_k + stage * ATT_TILE_BYTES));
#pragma unroll
    for (int kk = 0; kk < ATT_HD / 16; ++kk) wgmma_ss_n128(s, dq + 2 * kk, dk + 2 * kk, kk != 0 ? 1u : 0u);
    wgmma_commit();
  };
  // O += P.V of the tile in `stage`: one wgmma group.  The S fragment of columns [16 kk, 16 kk + 16) is exactly the A
  // fragment of k step kk, so P stays in registers.  The caller fences.
  auto issue_pv = [&](const uint32_t (&pa)[ATT_BN / 16][4], int stage) {
    const uint32_t sv = smem_u32(smem_v + stage * ATT_TILE_BYTES);
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk) {
      // V tile [128 kv x 64 hd], 128-byte rows: MN-major, 8-row k groups 1024 B apart, 16 kv rows (2048 B) per MMA
      const uint64_t dv = make_smem_desc(sv + kk * 2048, ATT_BN * 128, 1024);
      wgmma_rs_n64_tb(o, pa[kk], dv);
    }
    wgmma_commit();
  };
  // the element mask of kv tile kt on an S tile flagged partial
  auto mask_tile = [&](float (&s)[64], int kt) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int kv = kt * ATT_BN + 8 * i + 2 * t4 + e;
        int sk = 0x7fffffff, tk = 0x7fffffff;   // outside the sequence: matches no row
        if (kv < a.seq) {
          sk = __ldg(sg + kv);
          tk = __ldg(tm + kv);
        }
        if (!(sk == seg_q[0] && tk <= time_q[0])) s[4 * i + e] = -INFINITY;
        if (!(sk == seg_q[1] && tk <= time_q[1])) s[4 * i + 2 + e] = -INFINITY;
      }
    }
  };
  // online softmax of one S tile on the fragments, in place: s becomes P (fp32), m_run / l_run advance, alpha rescales O.
  // Row max over the thread's columns as a tree (4 dependent steps after the pairs instead of 16; max is exact, so any order
  // gives the same value), then over the 4 threads of the row.
  auto softmax = [&](float (&s)[64], float (&alpha)[2]) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float m16[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) m16[i] = fmaxf(s[4 * i + 2 * r], s[4 * i + 2 * r + 1]);
#pragma unroll
      for (int i = 0; i < 8; ++i) m16[i] = fmaxf(m16[i], m16[i + 8]);
#pragma unroll
      for (int i = 0; i < 4; ++i) m16[i] = fmaxf(m16[i], m16[i + 4]);
#pragma unroll
      for (int i = 0; i < 2; ++i) m16[i] = fmaxf(m16[i], m16[i + 2]);
      float mx = fmaxf(m16[0], m16[1]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[r], mx);
      // m_new == -inf: every score so far is masked, the reference is 0 and nothing is rescaled
      alpha[r] = (m_new == -INFINITY) ? 1.f : ex2_approx_f((m_run[r] - m_new) * c);
      m_run[r] = m_new;
      const float m_ref = (m_new == -INFINITY) ? 0.f : m_new * c;
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float p0 = ex2_approx_f(fmaf(s[4 * i + 2 * r], c, -m_ref));
        const float p1 = ex2_approx_f(fmaf(s[4 * i + 2 * r + 1], c, -m_ref));
        s[4 * i + 2 * r] = p0;
        s[4 * i + 2 * r + 1] = p1;
        sum += p0 + p1;
      }
      l_run[r] = l_run[r] * alpha[r] + sum;
    }
  };
  // The softmax is written out in both arms of the mask branch.  With one copy after the branch, ptxas waits for every
  // wgmma group where the arms join, that is before the softmax, and P(j-1).V(j-1) would no longer run under it.
  auto mask_and_softmax = [&](float (&s)[64], int entry, float (&alpha)[2]) {
    if (entry & 1) {
      mask_tile(s, entry >> 1);
      softmax(s, alpha);
    } else {
      softmax(s, alpha);
    }
  };
  // O *= alpha, then P -> the bf16 A fragments of the next P.V (all eight packed before it is issued back to back)
  auto rescale_and_pack = [&](const float (&alpha)[2], const float (&s)[64], uint32_t (&pa)[ATT_BN / 16][4]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i + 0] *= alpha[0];
      o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1];
      o[4 * i + 3] *= alpha[1];
    }
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk) {
      pa[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
    }
  };

  // Tensor-core turns: named barrier 1 + wg is this warpgroup's turn, 2 - wg the other's (256 threads: the two consumer
  // warpgroups).  A warpgroup issues its MMAs (S(0); S(j) and P(j-1).V(j-1); the last P.V) only in its turn and hands the
  // turn over right after issuing, so one warpgroup's softmax runs under the other's MMAs.  Warpgroup 0 takes the first
  // turn.  Both walk the same n_kv tiles, so both take n_kv + 1 turns, and every bar.sync meets one bar.arrive of the other
  // warpgroup: the first turn of warpgroup 0 meets the arrive below, every later turn the arrive after the other's previous
  // turn.  Warpgroup 1 makes no arrive after its last turn, where nothing would wait for it.  n_kv = 0 takes no turn.
  const int my_turn = 1 + wg, other_turn = 2 - wg;
  if (n_kv > 0) {
    float s[64];
    uint32_t pa[ATT_BN / 16][4];
    float alpha[2];
    if (wg == 1) named_bar_arrive(1, 256);

    // tile 0: S(0) alone
    mbar_wait(&k_full[0], 0);
    named_bar_sync(my_turn, 256);
    wgmma_fence();
    issue_qk(s, 0);
    named_bar_arrive(other_turn, 256);
    wgmma_wait<0>();
    wgmma_reg_fence(s);
    if (lane == 0) mbar_arrive(&k_empty[0]);
    mask_and_softmax(s, sched[1], alpha);
    rescale_and_pack(alpha, s, pa);

    // tile j: S(j) and P(j-1).V(j-1) in flight together; the softmax of tile j runs under P(j-1).V(j-1).  O is rescaled by
    // alpha(j) after P(j-1).V(j-1) has been added, then P(j).V(j) is added in the next turn: the same operations in the same
    // order as one tile at a time, so the same bits.
    int st = 0;          // stage of tile j - 1
    uint32_t ph = 0;
    for (int j = 1; j < n_kv; ++j) {
      const int kst = (st + 1 == ATT_STAGES) ? 0 : st + 1;
      const uint32_t kph = (kst == 0) ? ph ^ 1 : ph;
      mbar_wait(&k_full[kst], kph);
      mbar_wait(&v_full[st], ph);
      named_bar_sync(my_turn, 256);
      wgmma_reg_fence(o);
      wgmma_fence();
      issue_qk(s, kst);
      issue_pv(pa, st);
      named_bar_arrive(other_turn, 256);
      wgmma_wait<1>();   // S(j) has retired; P(j-1).V(j-1) may still run
      wgmma_reg_fence(s);
      if (lane == 0) mbar_arrive(&k_empty[kst]);
      mask_and_softmax(s, sched[1 + j], alpha);
      wgmma_wait<0>();
      wgmma_reg_fence(o);
      if (lane == 0) mbar_arrive(&v_empty[st]);
      rescale_and_pack(alpha, s, pa);
      st = kst;
      ph = kph;
    }

    // the last P.V
    mbar_wait(&v_full[st], ph);
    named_bar_sync(my_turn, 256);
    wgmma_reg_fence(o);
    wgmma_fence();
    issue_pv(pa, st);
    if (wg == 0) named_bar_arrive(other_turn, 256);
    wgmma_wait<0>();
    wgmma_reg_fence(o);
    if (lane == 0) mbar_arrive(&v_empty[st]);
  }

  // ---- epilogue: O / l -> bf16 -> out[b, qpos, h*64 + ...]
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = (l > 0.f) ? 1.f / l : 0.f;
    const int qpos = qt * ATT_BM + row0 + 8 * r;
    if (qpos >= a.seq) continue;
    if constexpr (kLse) {
      // lse = scale * max + ln(sum exp(scale * (s - max))) = ln 2 * (max * scale * log2 e + log2 l); +inf for a row without an
      // allowed score, so that the backward's exp(s * scale - lse) is 0 there
      if (t4 == 0) a.lse[static_cast<size_t>(bh) * a.seq + qpos] = (l > 0.f) ? (m_run[r] * c + log2f(l)) * 0.6931471805599453f : INFINITY;
    }
    __nv_bfloat16* dst;
    if (a.peer_count > 1) {
      const int pr = qpos / a.peer_chunk_rows;
      dst = a.peer_out[pr] + static_cast<size_t>(qpos - pr * a.peer_chunk_rows) * a.ldo + a.peer_col_begin + h * ATT_HD;
    } else {
      dst = a.out + (static_cast<size_t>(b) * a.seq + qpos) * a.ldo + h * ATT_HD;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i + 2 * t4) = pack_bf16x2(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
  }
}

int warmup_attn_bwd();

int warmup_attn() {
  int rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_fwd_kernel<false>), ATT_SMEM_BYTES, "attn_fwd_kernel");
  if (!rc) rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_fwd_kernel<true>), ATT_SMEM_BYTES, "attn_fwd_kernel<lse>");
  if (!rc) rc = warmup_attn_bwd();
  return rc;
}

}  // namespace pf

extern "C" int pf_attn_build_schedule(const int32_t* seg, const int32_t* time, int32_t batch, int32_t seq,
                                      int32_t* out, int64_t* allowed_pairs) {
  using namespace pf;
  PF_REQUIRE(batch > 0 && seq > 0, "pf_attn_build_schedule: bad shape");
  const int tiles = (seq + 127) / 128;
  const int stride = 1 + tiles;
  if (out == nullptr) return stride;
  PF_REQUIRE(seg && time, "pf_attn_build_schedule: null ids");
  for (int b = 0; b < batch; ++b) {
    const int32_t* sg = seg + static_cast<size_t>(b) * seq;
    const int32_t* tm = time + static_cast<size_t>(b) * seq;
    std::vector<int32_t> tmin(tiles), tmax(tiles), smin(tiles), smax(tiles);
    for (int t = 0; t < tiles; ++t) {
      const int lo = t * 128, hi = std::min(seq, lo + 128);
      int32_t a = tm[lo], bq = tm[lo], c = sg[lo], d = sg[lo];
      for (int i = lo; i < hi; ++i) {
        a = std::min(a, tm[i]);
        bq = std::max(bq, tm[i]);
        c = std::min(c, sg[i]);
        d = std::max(d, sg[i]);
      }
      tmin[t] = a; tmax[t] = bq; smin[t] = c; smax[t] = d;
    }
    int64_t pairs = 0;
    for (int qt = 0; qt < tiles; ++qt) {
      int32_t* row = out + (static_cast<size_t>(b) * tiles + qt) * stride;
      int cnt = 0;
      const int qlo = qt * 128, qhi = std::min(seq, qlo + 128);
      for (int kt = 0; kt < tiles; ++kt) {
        const int klo = kt * 128, khi = std::min(seq, klo + 128);
        if (tmax[qt] < tmin[kt]) continue;                              // no time-compatible pair
        if (smax[qt] < smin[kt] || smax[kt] < smin[qt]) continue;       // disjoint segment ranges
        const bool uniform = (smin[qt] == smax[qt]) && (smin[kt] == smax[kt]) && (smin[qt] == smin[kt]);
        const bool full = uniform && (tmin[qt] >= tmax[kt]) && (khi - klo == 128);
        int64_t n_allowed = 0;
        if (full) {
          n_allowed = static_cast<int64_t>(qhi - qlo) * (khi - klo);
        } else {
          for (int i = qlo; i < qhi; ++i)
            for (int j = klo; j < khi; ++j) n_allowed += (sg[i] == sg[j] && tm[i] >= tm[j]) ? 1 : 0;
          if (n_allowed == 0) continue;
        }
        pairs += n_allowed;
        row[1 + cnt] = (kt << 1) | (full ? 0 : 1);
        ++cnt;
      }
      row[0] = cnt;
      for (int i = 1 + cnt; i < stride; ++i) row[i] = 0;
    }
    if (allowed_pairs) allowed_pairs[b] = pairs;
  }
  return stride;
}

extern "C" int pf_attn_fwd_masked(const pf_attn_desc* d, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(d && d->q && d->k && d->v && (d->out || d->peer_count > 1) && d->seg && d->time && d->tile_sched, "pf_attn_fwd_masked: null pointer");
  PF_REQUIRE(d->head_dim == ATT_HD, "pf_attn_fwd_masked: head_dim %d unsupported (64 only)", d->head_dim);
  PF_REQUIRE(d->batch > 0 && d->heads > 0 && d->seq > 0, "pf_attn_fwd_masked: bad shape");
  const int q_tiles = (d->seq + ATT_BM - 1) / ATT_BM;
  PF_REQUIRE(d->sched_stride >= 1 + q_tiles, "pf_attn_fwd_masked: schedule stride %d too small", d->sched_stride);
  PF_REQUIRE(d->q_row_begin >= 0 && d->q_row_begin % ATT_BM == 0 && d->q_row_begin < d->seq,
             "pf_attn_fwd_masked: q_row_begin %d must be a multiple of %d inside the sequence", d->q_row_begin, ATT_BM);
  PF_REQUIRE(d->ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(d->out) & 15) == 0, "pf_attn_fwd_masked: out must be 16-byte aligned");
  // Every variant value runs the one kernel of this file; the values that name a q-tile grouping still require the schedule
  // they were defined with, so a caller's plan stays checked.
  PF_REQUIRE(d->variant == 0x10 || d->variant == 0x20 || (d->variant >= 0 && d->variant <= 3), "pf_attn_fwd_masked: bad variant 0x%x", d->variant);
  if (d->variant == 0x20)
    PF_REQUIRE(d->group_sched != nullptr && d->group_mask_index != nullptr && d->group_mask_bits != nullptr,
               "pf_attn_fwd_masked: variant 0x%x needs group_sched, group_mask_index and group_mask_bits", d->variant);
  if (d->variant == 0x10)
    PF_REQUIRE(d->pair_sched != nullptr && d->pair_mask_index != nullptr && d->pair_mask_bits != nullptr,
               "pf_attn_fwd_masked: variant 0x%x needs pair_sched, pair_mask_index and pair_mask_bits", d->variant);
  if (d->peer_count > 1) {
    PF_REQUIRE(d->batch == 1 && d->peer_count <= PF_MAX_PEERS && d->peer_chunk_rows > 0 &&
                   static_cast<long long>(d->peer_chunk_rows) * d->peer_count >= d->seq && d->peer_col_begin % 8 == 0,
               "pf_attn_fwd_masked: bad peer layout (batch %d, count %d, chunk rows %d, seq %d)", d->batch, d->peer_count,
               d->peer_chunk_rows, d->seq);
    // a rank's head group ends inside the row: past ldo the stores would land in the next row's columns
    PF_REQUIRE(d->peer_col_begin >= 0 && d->peer_col_begin + static_cast<long long>(d->heads) * ATT_HD <= d->ldo,
               "pf_attn_fwd_masked: peer columns [%d, %lld) exceed the row stride ldo %lld", d->peer_col_begin,
               d->peer_col_begin + static_cast<long long>(d->heads) * ATT_HD, static_cast<long long>(d->ldo));
    for (int i = 0; i < d->peer_count; ++i) {
      PF_REQUIRE(d->peer_out[i] != nullptr, "pf_attn_fwd_masked: peer_out[%d] is null", i);
      PF_REQUIRE((reinterpret_cast<uintptr_t>(d->peer_out[i]) & 15) == 0, "pf_attn_fwd_masked: peer_out[%d] must be 16-byte aligned", i);
    }
  }
  if (d->lse != nullptr)
    PF_REQUIRE(d->peer_count <= 1 && d->q_row_begin == 0,
               "pf_attn_fwd_masked: lse is computed for whole local launches only (peer_count %d, q_row_begin %d)", d->peer_count,
               d->q_row_begin);
  CUtensorMap tm[3];
  const void* ptrs[3] = {d->q, d->k, d->v};
  for (int i = 0; i < 3; ++i) {
    const uint64_t dims[3] = {ATT_HD, static_cast<uint64_t>(d->seq), static_cast<uint64_t>(d->batch) * d->heads};
    const uint64_t strides[2] = {ATT_HD * 2, static_cast<uint64_t>(d->seq) * ATT_HD * 2};
    const uint32_t box[3] = {ATT_HD, ATT_BN, 1};
    int rc = encode_tensor_map(&tm[i], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, ptrs[i], dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  AttnArgs a{};
  a.out = static_cast<__nv_bfloat16*>(d->out);
  a.ldo = d->ldo;
  a.batch = d->batch;
  a.heads = d->heads;
  a.seq = d->seq;
  a.q_tiles = q_tiles;
  a.scale_log2 = d->scale * 1.4426950408889634f;
  a.seg = d->seg;
  a.time = d->time;
  a.sched = d->tile_sched;
  a.sched_stride = d->sched_stride;
  a.peer_count = d->peer_count;
  a.peer_chunk_rows = d->peer_chunk_rows;
  a.peer_col_begin = d->peer_col_begin;
  for (int i = 0; i < PF_MAX_PEERS; ++i) a.peer_out[i] = static_cast<__nv_bfloat16*>(d->peer_out[i]);
  a.lse = d->lse;

  if (int rc = warmup_attn()) return rc;
  // q tile index = q_tiles - 1 - blockIdx.x: a shorter grid.x drops the leading (lowest) q tiles
  dim3 grid(q_tiles - d->q_row_begin / ATT_BM, d->heads, d->batch);
  if (a.lse != nullptr)
    attn_fwd_kernel<true><<<grid, ATT_THREADS, ATT_SMEM_BYTES, stream>>>(tm[0], tm[1], tm[2], a);
  else
    attn_fwd_kernel<false><<<grid, ATT_THREADS, ATT_SMEM_BYTES, stream>>>(tm[0], tm[1], tm[2], a);
  return check_launch("pf_attn_fwd_masked");
}
