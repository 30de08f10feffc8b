// pf_attn_bwd.cu — backward of the masked joint attention (pf_attn.cu) on Hopper warpgroup MMA (head_dim 64).
//
//   P = exp(scale * Q K^T - lse) on the allowed pairs, mask = (seg_q == seg_kv) && (time_q >= time_kv), 0 elsewhere
//   dV = P^T dO,   dS = P o (dO V^T - delta),   delta = rowsum(dO o O),   dQ = scale * dS K,   dK = scale * dS^T Q
//
// replaces the autograd backward of F.scaled_dot_product_attention with the dense [B,1,S,S] bool mask in the reference's
// training path (B:363-365, B:596-598; mask F:341-350).  Like the forward, only the tiles of the host-built schedules are
// visited and the element mask is evaluated from seg / time on the tiles flagged partial.  Three launches, no atomics:
//   attn_bwd_delta_kernel   one warp per (b, h, row): delta = sum_d dO o O in fp32
//   attn_bwd_dkdv_kernel    one CTA per (b, h, 128-row kv tile); K and V loaded once, the q tiles of the kv schedule stream
//                           Q and dO through a 2-stage mbarrier ring.  Per q tile each consumer warpgroup (64 kv rows)
//                           computes S^T = K Q^T and dP^T = V dO^T (wgmma, smem operands), P^T and dS^T on the fragments,
//                           then dV += P^T dO and dK += dS^T Q with P^T / dS^T re-packed in registers as the bf16 A operand
//                           and Q / dO read MN-major from the same tiles.
//   attn_bwd_dq_kernel      one CTA per (b, h, 128-row q tile) on the forward's schedule; Q and dO loaded once, K and V
//                           streamed.  S = Q K^T, dP = dO V^T, dS on the fragments, dQ += dS K (A from registers).
// Register budget: the 128-wide streamed tile is consumed in two halves of 64 columns, so a consumer thread holds S and dP
// as 32 + 32 fp32 (plus dK and dV, 32 + 32, in the kv-major pass) instead of 64 + 64: no spills under the 232-register cap.
#include <vector>

#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

constexpr int BWD_BM = 128;       // rows of the CTA's own tile (kv rows in the dK/dV pass, q rows in the dQ pass)
constexpr int BWD_BN = 128;       // rows of a streamed tile
constexpr int BWD_HALF = 64;      // streamed columns per MMA round
constexpr int BWD_HD = 64;
constexpr int BWD_STAGES = 2;
constexpr int BWD_THREADS = 384;
constexpr int BWD_TILE_BYTES = 128 * BWD_HD * 2;   // 16 KB: one [128 x 64] bf16 tile, 128-byte rows, SWIZZLE_128B
constexpr int BWD_SMEM_BYTES = (2 + 2 * BWD_STAGES) * BWD_TILE_BYTES + 1024;
constexpr float LOG2E = 1.4426950408889634f;

struct AttnBwdArgs {
  int batch, heads, seq, tiles;
  float scale, scale_log2;
  const int* seg;
  const int* time;
  const int* sched;       // q-major (dQ pass) or kv-major (dK/dV pass)
  int sched_stride;
  const float* lse;
  const float* delta;
  __nv_bfloat16* d0;      // dK (dK/dV pass) or dQ (dQ pass)
  __nv_bfloat16* d1;      // dV (dK/dV pass)
};

// delta[b, h, s] = sum_d dO[b, s, h*64 + d] * O[b, s, h*64 + d]: one warp per row, two columns per lane.
__global__ void __launch_bounds__(256) attn_bwd_delta_kernel(const __nv_bfloat16* __restrict__ out, long long ldo, long long out_bs,
                                                             const __nv_bfloat16* __restrict__ dout, long long lddo, long long dout_bs,
                                                             float* __restrict__ delta, int heads, int seq, long long rows) {
  const long long row = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int s = static_cast<int>(row % seq);
  const long long bh = row / seq;
  const int h = static_cast<int>(bh % heads);
  const long long b = bh / heads;
  const __nv_bfloat162 o = *reinterpret_cast<const __nv_bfloat162*>(out + b * out_bs + s * ldo + h * BWD_HD + 2 * lane);
  const __nv_bfloat162 g = *reinterpret_cast<const __nv_bfloat162*>(dout + b * dout_bs + s * lddo + h * BWD_HD + 2 * lane);
  float acc = __low2float(o) * __low2float(g) + __high2float(o) * __high2float(g);
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
  if (lane == 0) delta[row] = acc;
}

// Store a [64 x 64] fp32 accumulator fragment (rows row0, row0 + 8 of the thread) as bf16 rows of a [.., seq, 64] tensor.
__device__ __forceinline__ void bwd_store_rows(__nv_bfloat16* base, int row0, int seq, const float (&acc)[32], float mul) {
  const int t4 = threadIdx.x & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int pos = row0 + 8 * r;
    if (pos >= seq) continue;
    __nv_bfloat16* dst = base + static_cast<size_t>(pos) * BWD_HD;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i + 2 * t4) = pack_bf16x2(acc[4 * i + 2 * r] * mul, acc[4 * i + 2 * r + 1] * mul);
  }
}

// The A fragments of k steps kk = 0..3 of a [64 x 64] fp32 accumulator, as bf16 (the fragment of columns [16 kk, 16 kk + 16)
// is exactly the A fragment of k step kk).
__device__ __forceinline__ void bwd_pack_a(const float (&x)[32], uint32_t (&pa)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    pa[kk][0] = pack_bf16x2(x[8 * kk + 0], x[8 * kk + 1]);
    pa[kk][1] = pack_bf16x2(x[8 * kk + 2], x[8 * kk + 3]);
    pa[kk][2] = pack_bf16x2(x[8 * kk + 4], x[8 * kk + 5]);
    pa[kk][3] = pack_bf16x2(x[8 * kk + 6], x[8 * kk + 7]);
  }
}

// acc[64 x 64] += A (registers, k = 64 rows of the smem tile) * tile rows [row_off, row_off + 64) read MN-major
__device__ __forceinline__ void bwd_mma_rs(float (&acc)[32], const uint32_t (&pa)[4][4], uint32_t tile_saddr, int row_off) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    // [k rows x 64 hd] with 128-byte rows: MN-major, 8-row k groups 1024 B apart, 16 k rows (2048 B) per MMA
    const uint64_t db = make_smem_desc(tile_saddr + (row_off + 16 * kk) * 128, 128 * 128, 1024);
    wgmma_rs_n64_tb(acc, pa[kk], db);
  }
}

// ===================================================================================================================
// dK / dV: CTA = (kv tile, h, b).  Producer: K, V once; then (Q, dO) of every q tile of the kv schedule row.
// Consumer thread (warp w of warpgroup wg, g = lane / 4, t = lane % 4) owns kv rows 64 wg + 16 w + g (+ 8) and, in each
// 64-column half of a q tile, q columns 8 i + 2 t (+ 1), i < 8.
// ===================================================================================================================
__global__ void __launch_bounds__(BWD_THREADS, 1)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                     const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_do, const AttnBwdArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_k = smem;
  uint8_t* smem_v = smem + BWD_TILE_BYTES;
  uint8_t* smem_q = smem + 2 * BWD_TILE_BYTES;                       // stage st: smem_q + st * TILE
  uint8_t* smem_do = smem_q + BWD_STAGES * BWD_TILE_BYTES;

  __shared__ __align__(8) uint64_t bar_kv;
  __shared__ __align__(8) uint64_t full[BWD_STAGES], empty[BWD_STAGES];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wgroup = warp >> 2;
  const int kt = blockIdx.x;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int bh = b * a.heads + h;
  const int* sched = a.sched + (static_cast<size_t>(b) * a.tiles + kt) * a.sched_stride;
  const int n_q = sched[0];

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    tma_prefetch_desc(&tm_do);
    mbar_init(&bar_kv, 1);
    for (int i = 0; i < BWD_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wgroup == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      mbar_arrive_expect_tx(&bar_kv, 2 * BWD_TILE_BYTES);
      tma_load_3d(smem_k, &tm_k, &bar_kv, 0, kt * BWD_BM, bh);
      tma_load_3d(smem_v, &tm_v, &bar_kv, 0, kt * BWD_BM, bh);
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < n_q; ++j) {
        const int qt = sched[1 + j] >> 1;
        mbar_wait(&empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&full[st], 2 * BWD_TILE_BYTES);
        tma_load_3d(smem_q + st * BWD_TILE_BYTES, &tm_q, &full[st], 0, qt * BWD_BN, bh);
        tma_load_3d(smem_do + st * BWD_TILE_BYTES, &tm_do, &full[st], h * BWD_HD, qt * BWD_BN, b);
        if (++st == BWD_STAGES) {
          st = 0;
          ph ^= 1;
        }
      }
    }
    return;
  }

  setmaxnreg_inc<232>();
  const int wg = wgroup - 1;
  const int g4 = lane >> 2, t4 = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + g4;
  const float c = a.scale_log2;
  const int* sg = a.seg + static_cast<size_t>(b) * a.seq;
  const int* tmv = a.time + static_cast<size_t>(b) * a.seq;
  const float* lse = a.lse + static_cast<size_t>(bh) * a.seq;
  const float* dlt = a.delta + static_cast<size_t>(bh) * a.seq;
  int seg_k[2], time_k[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int kv = kt * BWD_BM + row0 + 8 * r;
    const bool ok = kv < a.seq;
    seg_k[r] = ok ? sg[kv] : 0x7fffffff;        // a kv row past the sequence matches no q column
    time_k[r] = ok ? tmv[kv] : 0x7fffffff;
  }
  const bool kv_tail = (kt + 1) * BWD_BM > a.seq;
  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dk[i] = dv[i] = 0.f;

  mbar_wait(&bar_kv, 0);
  const uint64_t dk_desc = make_smem_desc_kmajor_sw128(smem_u32(smem_k) + wg * (64 * 128));
  const uint64_t dv_desc = make_smem_desc_kmajor_sw128(smem_u32(smem_v) + wg * (64 * 128));
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < n_q; ++j) {
    const int entry = sched[1 + j];
    const int qt = entry >> 1;
    const bool masked = (entry & 1) != 0 || kv_tail || (qt + 1) * BWD_BN > a.seq;
    const uint32_t sq = smem_u32(smem_q + st * BWD_TILE_BYTES);
    const uint32_t sdo = smem_u32(smem_do + st * BWD_TILE_BYTES);
    mbar_wait(&full[st], ph);
#pragma unroll 1
    for (int hf = 0; hf < 2; ++hf) {
      // ---- S^T = K Q^T and dP^T = V dO^T over the 64 q columns of this half
      float s[32], dp[32];
      {
        const uint64_t bq = make_smem_desc_kmajor_sw128(sq + hf * (64 * 128));
        const uint64_t bdo = make_smem_desc_kmajor_sw128(sdo + hf * (64 * 128));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BWD_HD / 16; ++kk) wgmma_ss_n64(s, dk_desc + 2 * kk, bq + 2 * kk, kk != 0 ? 1u : 0u);
#pragma unroll
        for (int kk = 0; kk < BWD_HD / 16; ++kk) wgmma_ss_n64(dp, dv_desc + 2 * kk, bdo + 2 * kk, kk != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(s);
        wgmma_reg_fence(dp);
      }
      // ---- P^T = exp2(s c - lse log2 e), dS^T = P^T (dP^T - delta); column q = qt*128 + hf*64 + 8 i + 2 t + e
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int q = qt * BWD_BN + hf * BWD_HALF + 8 * i + 2 * t4 + e;
          const bool q_ok = q < a.seq;
          const float l2 = q_ok ? __ldg(lse + q) * LOG2E : INFINITY;
          const float dl = q_ok ? __ldg(dlt + q) : 0.f;
          float p0 = ex2_approx_f(fmaf(s[4 * i + e], c, -l2));
          float p1 = ex2_approx_f(fmaf(s[4 * i + 2 + e], c, -l2));
          if (masked) {
            int sqv = -0x7fffffff, tqv = -0x7fffffff;   // a q column past the sequence matches no kv row
            if (q_ok) {
              sqv = __ldg(sg + q);
              tqv = __ldg(tmv + q);
            }
            if (!(sqv == seg_k[0] && time_k[0] <= tqv)) p0 = 0.f;
            if (!(sqv == seg_k[1] && time_k[1] <= tqv)) p1 = 0.f;
          }
          s[4 * i + e] = p0;
          s[4 * i + 2 + e] = p1;
          dp[4 * i + e] = p0 * (dp[4 * i + e] - dl);
          dp[4 * i + 2 + e] = p1 * (dp[4 * i + 2 + e] - dl);
        }
      }
      // ---- dV += P^T dO, dK += dS^T Q (k = the 64 q rows of this half)
      uint32_t pa[4][4], da[4][4];
      bwd_pack_a(s, pa);
      bwd_pack_a(dp, da);
      wgmma_reg_fence(dv);
      wgmma_reg_fence(dk);
      wgmma_fence();
      bwd_mma_rs(dv, pa, sdo, hf * 64);
      bwd_mma_rs(dk, da, sq, hf * 64);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(dv);
      wgmma_reg_fence(dk);
    }
    if (lane == 0) mbar_arrive(&empty[st]);
    if (++st == BWD_STAGES) {
      st = 0;
      ph ^= 1;
    }
  }

  const size_t base = static_cast<size_t>(bh) * a.seq * BWD_HD;
  bwd_store_rows(a.d0 + base, kt * BWD_BM + row0, a.seq, dk, a.scale);
  bwd_store_rows(a.d1 + base, kt * BWD_BM + row0, a.seq, dv, 1.f);
}

// ===================================================================================================================
// dQ: CTA = (q tile, h, b), heavy (late) q tiles first.  Producer: Q, dO once; then (K, V) of every kv tile of the row.
// Consumer thread owns q rows 64 wg + 16 w + g (+ 8) and, in each 64-column half of a kv tile, kv columns 8 i + 2 t (+ 1).
// ===================================================================================================================
__global__ void __launch_bounds__(BWD_THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                   const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_do, const AttnBwdArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_do = smem + BWD_TILE_BYTES;
  uint8_t* smem_k = smem + 2 * BWD_TILE_BYTES;
  uint8_t* smem_v = smem_k + BWD_STAGES * BWD_TILE_BYTES;

  __shared__ __align__(8) uint64_t bar_q;
  __shared__ __align__(8) uint64_t full[BWD_STAGES], empty[BWD_STAGES];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wgroup = warp >> 2;
  const int qt = a.tiles - 1 - static_cast<int>(blockIdx.x);
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int bh = b * a.heads + h;
  const int* sched = a.sched + (static_cast<size_t>(b) * a.tiles + qt) * a.sched_stride;
  const int n_kv = sched[0];

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    tma_prefetch_desc(&tm_do);
    mbar_init(&bar_q, 1);
    for (int i = 0; i < BWD_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wgroup == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      mbar_arrive_expect_tx(&bar_q, 2 * BWD_TILE_BYTES);
      tma_load_3d(smem_q, &tm_q, &bar_q, 0, qt * BWD_BM, bh);
      tma_load_3d(smem_do, &tm_do, &bar_q, h * BWD_HD, qt * BWD_BM, b);
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < n_kv; ++j) {
        const int kt = sched[1 + j] >> 1;
        mbar_wait(&empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&full[st], 2 * BWD_TILE_BYTES);
        tma_load_3d(smem_k + st * BWD_TILE_BYTES, &tm_k, &full[st], 0, kt * BWD_BN, bh);
        tma_load_3d(smem_v + st * BWD_TILE_BYTES, &tm_v, &full[st], 0, kt * BWD_BN, bh);
        if (++st == BWD_STAGES) {
          st = 0;
          ph ^= 1;
        }
      }
    }
    return;
  }

  setmaxnreg_inc<232>();
  const int wg = wgroup - 1;
  const int g4 = lane >> 2, t4 = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + g4;
  const float c = a.scale_log2;
  const int* sg = a.seg + static_cast<size_t>(b) * a.seq;
  const int* tmv = a.time + static_cast<size_t>(b) * a.seq;
  int seg_q[2], time_q[2];
  float l2[2], dl[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = qt * BWD_BM + row0 + 8 * r;
    const bool ok = q < a.seq;
    seg_q[r] = ok ? sg[q] : -0x7fffffff;        // a q row past the sequence matches no kv column
    time_q[r] = ok ? tmv[q] : -0x7fffffff;
    l2[r] = ok ? a.lse[static_cast<size_t>(bh) * a.seq + q] * LOG2E : INFINITY;
    dl[r] = ok ? a.delta[static_cast<size_t>(bh) * a.seq + q] : 0.f;
  }
  const bool q_tail = (qt + 1) * BWD_BM > a.seq;
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;

  mbar_wait(&bar_q, 0);
  const uint64_t aq = make_smem_desc_kmajor_sw128(smem_u32(smem_q) + wg * (64 * 128));
  const uint64_t ado = make_smem_desc_kmajor_sw128(smem_u32(smem_do) + wg * (64 * 128));
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < n_kv; ++j) {
    const int entry = sched[1 + j];
    const int kt = entry >> 1;
    const bool masked = (entry & 1) != 0 || q_tail || (kt + 1) * BWD_BN > a.seq;
    const uint32_t sk = smem_u32(smem_k + st * BWD_TILE_BYTES);
    const uint32_t sv = smem_u32(smem_v + st * BWD_TILE_BYTES);
    mbar_wait(&full[st], ph);
#pragma unroll 1
    for (int hf = 0; hf < 2; ++hf) {
      float s[32], dp[32];
      {
        const uint64_t bk = make_smem_desc_kmajor_sw128(sk + hf * (64 * 128));
        const uint64_t bv = make_smem_desc_kmajor_sw128(sv + hf * (64 * 128));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BWD_HD / 16; ++kk) wgmma_ss_n64(s, aq + 2 * kk, bk + 2 * kk, kk != 0 ? 1u : 0u);
#pragma unroll
        for (int kk = 0; kk < BWD_HD / 16; ++kk) wgmma_ss_n64(dp, ado + 2 * kk, bv + 2 * kk, kk != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(s);
        wgmma_reg_fence(dp);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float p0 = ex2_approx_f(fmaf(s[4 * i + e], c, -l2[0]));
          float p1 = ex2_approx_f(fmaf(s[4 * i + 2 + e], c, -l2[1]));
          if (masked) {
            const int kv = kt * BWD_BN + hf * BWD_HALF + 8 * i + 2 * t4 + e;
            int skv = 0x7fffffff, tkv = 0x7fffffff;   // a kv column past the sequence matches no q row
            if (kv < a.seq) {
              skv = __ldg(sg + kv);
              tkv = __ldg(tmv + kv);
            }
            if (!(skv == seg_q[0] && tkv <= time_q[0])) p0 = 0.f;
            if (!(skv == seg_q[1] && tkv <= time_q[1])) p1 = 0.f;
          }
          dp[4 * i + e] = p0 * (dp[4 * i + e] - dl[0]);
          dp[4 * i + 2 + e] = p1 * (dp[4 * i + 2 + e] - dl[1]);
        }
      }
      uint32_t da[4][4];
      bwd_pack_a(dp, da);
      wgmma_reg_fence(dq);
      wgmma_fence();
      bwd_mma_rs(dq, da, sk, hf * 64);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(dq);
    }
    if (lane == 0) mbar_arrive(&empty[st]);
    if (++st == BWD_STAGES) {
      st = 0;
      ph ^= 1;
    }
  }
  bwd_store_rows(a.d0 + static_cast<size_t>(bh) * a.seq * BWD_HD, qt * BWD_BM + row0, a.seq, dq, a.scale);
}

int warmup_attn_bwd() {
  int rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_dkdv_kernel), BWD_SMEM_BYTES, "attn_bwd_dkdv_kernel");
  if (!rc) rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_bwd_dq_kernel), BWD_SMEM_BYTES, "attn_bwd_dq_kernel");
  return rc;
}

}  // namespace pf

extern "C" int pf_attn_bwd_masked(const pf_attn_bwd_desc* d, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(d && d->q && d->k && d->v && d->out && d->dout && d->lse && d->seg && d->time && d->tile_sched && d->kv_sched &&
                 d->delta && d->dq && d->dk && d->dv,
             "pf_attn_bwd_masked: null pointer");
  PF_REQUIRE(d->head_dim == BWD_HD, "pf_attn_bwd_masked: head_dim %d unsupported (64 only)", d->head_dim);
  PF_REQUIRE(d->batch > 0 && d->heads > 0 && d->seq > 0, "pf_attn_bwd_masked: bad shape");
  const int tiles = (d->seq + BWD_BM - 1) / BWD_BM;
  PF_REQUIRE(d->sched_stride >= 1 + tiles, "pf_attn_bwd_masked: schedule stride %d too small", d->sched_stride);
  PF_REQUIRE(d->ldo >= static_cast<int64_t>(d->heads) * BWD_HD && d->lddo >= static_cast<int64_t>(d->heads) * BWD_HD &&
                 d->ldo % 8 == 0 && d->lddo % 8 == 0 && (reinterpret_cast<uintptr_t>(d->out) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(d->dout) & 15) == 0,
             "pf_attn_bwd_masked: out / dout need row strides >= heads*64, multiples of 8, 16-byte aligned (ldo %lld, lddo %lld)",
             static_cast<long long>(d->ldo), static_cast<long long>(d->lddo));
  PF_REQUIRE(d->out_batch_stride > 0 && d->dout_batch_stride > 0 && d->out_batch_stride % 8 == 0 && d->dout_batch_stride % 8 == 0,
             "pf_attn_bwd_masked: out / dout batch strides must be positive multiples of 8 elements (out_batch_stride %lld, "
             "dout_batch_stride %lld)", static_cast<long long>(d->out_batch_stride), static_cast<long long>(d->dout_batch_stride));
  CUtensorMap tm[4];
  const void* ptrs[3] = {d->q, d->k, d->v};
  for (int i = 0; i < 3; ++i) {
    const uint64_t dims[3] = {BWD_HD, static_cast<uint64_t>(d->seq), static_cast<uint64_t>(d->batch) * d->heads};
    const uint64_t strides[2] = {BWD_HD * 2, static_cast<uint64_t>(d->seq) * BWD_HD * 2};
    const uint32_t box[3] = {BWD_HD, 128, 1};
    if (int rc = encode_tensor_map(&tm[i], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, ptrs[i], dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B))
      return rc;
  }
  {
    // dO [batch, seq, heads*64] with row stride lddo and batch stride dout_batch_stride: head h is the 64-column box at
    // column h*64
    const uint64_t dims[3] = {static_cast<uint64_t>(d->heads) * BWD_HD, static_cast<uint64_t>(d->seq), static_cast<uint64_t>(d->batch)};
    const uint64_t strides[2] = {static_cast<uint64_t>(d->lddo) * 2, static_cast<uint64_t>(d->dout_batch_stride) * 2};
    const uint32_t box[3] = {BWD_HD, 128, 1};
    if (int rc = encode_tensor_map(&tm[3], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, d->dout, dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B))
      return rc;
  }
  if (int rc = warmup_attn_bwd()) return rc;

  const long long rows = static_cast<long long>(d->batch) * d->heads * d->seq;
  attn_bwd_delta_kernel<<<static_cast<unsigned>((rows + 7) / 8), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(d->out), d->ldo, d->out_batch_stride, static_cast<const __nv_bfloat16*>(d->dout), d->lddo,
      d->dout_batch_stride, d->delta, d->heads,
      d->seq, rows);
  if (int rc = check_launch("pf_attn_bwd_masked (delta)")) return rc;

  AttnBwdArgs a{};
  a.batch = d->batch;
  a.heads = d->heads;
  a.seq = d->seq;
  a.tiles = tiles;
  a.scale = d->scale;
  a.scale_log2 = d->scale * LOG2E;
  a.seg = d->seg;
  a.time = d->time;
  a.sched_stride = d->sched_stride;
  a.lse = d->lse;
  a.delta = d->delta;
  const dim3 grid(tiles, d->heads, d->batch);

  a.sched = d->kv_sched;
  a.d0 = static_cast<__nv_bfloat16*>(d->dk);
  a.d1 = static_cast<__nv_bfloat16*>(d->dv);
  attn_bwd_dkdv_kernel<<<grid, BWD_THREADS, BWD_SMEM_BYTES, stream>>>(tm[0], tm[1], tm[2], tm[3], a);
  if (int rc = check_launch("pf_attn_bwd_masked (dk, dv)")) return rc;

  a.sched = d->tile_sched;
  a.d0 = static_cast<__nv_bfloat16*>(d->dq);
  a.d1 = nullptr;
  attn_bwd_dq_kernel<<<grid, BWD_THREADS, BWD_SMEM_BYTES, stream>>>(tm[0], tm[1], tm[2], tm[3], a);
  return check_launch("pf_attn_bwd_masked (dq)");
}
