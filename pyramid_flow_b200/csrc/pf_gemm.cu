// pf_gemm.cu — persistent warp-specialised bf16 GEMM on Hopper warpgroup MMA (wgmma) with fused epilogues.
//
//   out = epilogue(A[rows, K] . W[N, K]^T + bias)
//
// Three kernels, one CTA per SM (persistent, static tile schedule), 384 threads: warpgroup 0 (one lane) is the TMA producer
// (SWIZZLE_128B boxes, mbarrier tx-count), warpgroups 1 and 2 consume with wgmma.mma_async, fp32 accumulators in registers.
//   256 x 128 tiles in 2-CTA clusters (every step GEMM; 128 | N): each consumer warpgroup owns 128 rows (2 x m64n128k16 per
//       k16 step, 128 accumulators per thread); the W box is split between the two producers of a cluster and multicast into
//       both CTAs; the epilogue runs straight from the accumulator fragments.
//   128 x 128 and 128 x 64 tiles (pf_common.cuh "shared TMA -> wgmma pipeline"): each consumer warpgroup owns 64 rows; after
//       the K loop the fragments are staged through shared memory so that the epilogue runs with one thread per output row.
//       Taken for N not a multiple of 128, and when the wave-quantisation cost model prefers them (few rows).
// The producer runs ahead into the next tile's stages while the consumers are in the epilogue.
//
// Epilogues (include/pf_b200.h PF_EPI_*): bias / GELU-tanh / fp32 store / gate*x+residual / per-head RMSNorm + RoPE
// with head-major Q,K,V stores / the single-block fused q|k|v|mlp split; for the text encoders GEGLU (gate and linear
// columns 64 apart in every 128-wide tile, half-width output), quick-GELU and exact (erf) GELU.
// pf_gemm_fp8 runs the cluster kernel on e4m3 operands: 128 x 128 tiles (one 64-row half per consumer warpgroup), K = 128
// per stage, per-stage promotion of the fp8 partial sums into fp32, and the same epilogues after the per-row x per-column
// dequantisation scale.
// Reference op sites are listed in include/pf_b200.h at pf_gemm_bf16.
#include <cstdlib>

#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

struct GemmArgs {
  int batches, row_begin, row_count;
  int n, k;
  int m_tiles, n_tiles;
  const float* bias;
  void* out;
  long long ldo;
  int out_batch_rows, out_row_begin, out_col_begin;
  const float* gate;
  long long gate_batch_stride;
  __nv_bfloat16* q_out;
  __nv_bfloat16* k_out;
  __nv_bfloat16* v_out;
  const float* rope;
  const float* q_norm_w;
  const float* k_norm_w;
  float norm_eps;
  int heads, head_dim, seq_len;
  int n_split;
  // sequence parallel: q/k/v heads go straight into the owning rank's [3][peer_heads][peer_seq][64] buffer (pf_b200.h)
  __nv_bfloat16* peer_qkv[PF_MAX_PEERS];
  int peer_count, peer_heads, peer_seq, peer_row0;
  int epi_staged;   // 128-row kernels' GATE_RESID: whole-row read-modify-write, one warp per row segment (PF_OPT_GEMM_STAGED_RESID)
  // e4m3 operands (pf_gemm_fp8): a_scale[b * rows_per_batch + row_begin + m], w_scale[n]
  const float* a_scale;
  const float* w_scale;
  int rows_per_batch;
};

constexpr int BM = PIPE_BM;
constexpr int BK = PIPE_BK;

// Relative rates (FLOP/s) of the three kernels, for the wave-quantisation choice in pf_gemm_bf16.  tools/gemm_bench.py on an
// H100 80GB HBM3 (700 W power limit) at the step's full-size shapes (M = 30720 / 30976): 256 x 128 cluster 456 - 678 TFLOP/s,
// 1.21 - 1.44 x the 128 x 128 kernel (340 - 489); 128 x 64 0.72 - 0.85 x the 128 x 128 kernel.
constexpr double GEMM_RATE_CLUSTER = 1.25;
constexpr double GEMM_RATE_128 = 1.0;
constexpr double GEMM_RATE_64 = 0.75;

// the bf16-output activations of the single-column epilogues (GELU_BF16, QKV_GELU's mlp part, QUICK_GELU, GELU_ERF)
template <int EPI>
__device__ __forceinline__ float epi_act(float x) {
  if constexpr (EPI == PF_EPI_GELU_BF16 || EPI == PF_EPI_QKV_GELU) return gelu_tanh_f(x);
  if constexpr (EPI == PF_EPI_QUICK_GELU_BF16) return x * rcp_approx_f(1.0f + ex2_approx_f(-1.702f * 1.4426950408889634f * x));
  if constexpr (EPI == PF_EPI_GELU_ERF_BF16) return 0.5f * x * (1.0f + erff(x * 0.7071067811865476f));
  return x;
}
constexpr bool epi_is_act_bf16(int epi) {
  return epi == PF_EPI_GELU_BF16 || epi == PF_EPI_QUICK_GELU_BF16 || epi == PF_EPI_GELU_ERF_BF16;
}

// ---- epilogue helpers (one thread == one output row) -----------------------
__device__ __forceinline__ void store_bf16x32(__nv_bfloat16* dst, const float (&x)[32]) {
  uint4* d4 = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint4 u;
    u.x = pack_bf16x2(x[8 * i + 0], x[8 * i + 1]);
    u.y = pack_bf16x2(x[8 * i + 2], x[8 * i + 3]);
    u.z = pack_bf16x2(x[8 * i + 4], x[8 * i + 5]);
    u.w = pack_bf16x2(x[8 * i + 6], x[8 * i + 7]);
    d4[i] = u;
  }
}

// x[0..32) = staged accumulators + bias
__device__ __forceinline__ void load_bias32(float (&x)[32], const float* srow, const float* bias) {
  const float4* s4 = reinterpret_cast<const float4*>(srow);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = s4[i];
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias != nullptr) b = __ldg(reinterpret_cast<const float4*>(bias) + i);
    x[4 * i + 0] = v.x + b.x;
    x[4 * i + 1] = v.y + b.y;
    x[4 * i + 2] = v.z + b.z;
    x[4 * i + 3] = v.w + b.w;
  }
}

// One head (64 columns) of q / k / v for one token; `srow` = this token's staged accumulators at the head's first column.
// section 0 = q, 1 = k (RMSNorm over the head N:66-79, then RoPE B:34-39), 2 = v (plain store).
__device__ __forceinline__ void qkv_head_epilogue(const GemmArgs& g, const float* srow, int n0, int b, int pos, bool valid) {
  float x[64];
  {
    float lo[32], hi[32];
    load_bias32(lo, srow, g.bias ? g.bias + n0 : nullptr);
    load_bias32(hi, srow + 32, g.bias ? g.bias + n0 + 32 : nullptr);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      x[i] = lo[i];
      x[32 + i] = hi[i];
    }
  }
  const int inner = g.heads * g.head_dim;
  const int section = n0 / inner;
  const int head = (n0 - section * inner) / g.head_dim;
  __nv_bfloat16* base = section == 0 ? g.q_out : (section == 1 ? g.k_out : g.v_out);
  if (section < 2) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;   // four chains: a single 64-long FFMA chain is 256+ cycles of latency
#pragma unroll
    for (int i = 0; i < 64; i += 4) {
      s0 = fmaf(x[i + 0], x[i + 0], s0);
      s1 = fmaf(x[i + 1], x[i + 1], s1);
      s2 = fmaf(x[i + 2], x[i + 2], s2);
      s3 = fmaf(x[i + 3], x[i + 3], s3);
    }
    const float ss = (s0 + s1) + (s2 + s3);
    const float r = rsqrtf(ss * (1.0f / 64.0f) + g.norm_eps);
    const float4* w4 = reinterpret_cast<const float4*>(section == 0 ? g.q_norm_w : g.k_norm_w);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float4 w = __ldg(w4 + i);
      x[4 * i + 0] *= r * w.x;
      x[4 * i + 1] *= r * w.y;
      x[4 * i + 2] *= r * w.z;
      x[4 * i + 3] *= r * w.w;
    }
    if (g.rope != nullptr && valid) {
      const float4* cs4 = reinterpret_cast<const float4*>(g.rope + static_cast<size_t>(pos) * 64);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 cs = __ldg(cs4 + i);  // (cos_{2i}, sin_{2i}, cos_{2i+1}, sin_{2i+1})
        const float a0 = x[4 * i + 0], a1 = x[4 * i + 1], a2 = x[4 * i + 2], a3 = x[4 * i + 3];
        x[4 * i + 0] = cs.x * a0 - cs.y * a1;
        x[4 * i + 1] = cs.y * a0 + cs.x * a1;
        x[4 * i + 2] = cs.z * a2 - cs.w * a3;
        x[4 * i + 3] = cs.w * a2 + cs.z * a3;
      }
    }
  }
  if (valid) {
    __nv_bfloat16* dst;
    if (g.peer_count > 1) {
      const int r = head / g.peer_heads, hl = head - r * g.peer_heads;
      dst = g.peer_qkv[r] + ((static_cast<size_t>(section) * g.peer_heads + hl) * g.peer_seq + g.peer_row0 + pos) * 64;
    } else {
      dst = base + ((static_cast<size_t>(b) * g.heads + head) * g.seq_len + pos) * 64;
    }
    float lo[32], hi[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      lo[i] = x[i];
      hi[i] = x[32 + i];
    }
    store_bf16x32(dst, lo);
    store_bf16x32(dst + 32, hi);
  }
}

// Epilogue of one warpgroup's 64-row slice of the staged accumulator tile.  `tid` = thread index in the warpgroup: the
// row-per-thread forms give thread (row = tid % 64, half = tid / 64) every second 32-column chunk (or 64-column head) of its
// row; the whole-row GATE_RESID form gives each warp 16 rows and lets its lanes sweep a row's columns, so that the
// read-modify-write of the fp32 residual stream moves BN * 4 contiguous bytes per warp instruction.
template <int BN, int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmArgs& g, const float* acc_rows, int tid, int b, int m_base, int n_base) {
  constexpr int PITCH = PipeCfg<BN>::ACC_PITCH;
  const int row = tid & 63, half = tid >> 6;
  const int m = m_base + row;
  const bool valid = m < g.row_count;
  const size_t out_row = static_cast<size_t>(b) * g.out_batch_rows + g.out_row_begin + m;
  const float* srow = acc_rows + row * PITCH;
  bool qkv_tile = (EPI == PF_EPI_QKV_ROPE);
  if (EPI == PF_EPI_QKV_GELU) qkv_tile = n_base < g.n_split;

  if constexpr (EPI == PF_EPI_GEGLU_BF16) {
    // gate columns [32 half, +32) of the tile, linear columns 64 further; output columns n_base / 2 + 32 half + [0, 32)
    static_assert(BN == 128, "GEGLU runs on 128-wide tiles only");
    float x[32], lin[32];
    load_bias32(x, srow + 32 * half, g.bias ? g.bias + n_base + 32 * half : nullptr);
    load_bias32(lin, srow + 64 + 32 * half, g.bias ? g.bias + n_base + 64 + 32 * half : nullptr);
#pragma unroll
    for (int i = 0; i < 32; ++i) x[i] = gelu_tanh_f(x[i]) * lin[i];
    if (valid) store_bf16x32(reinterpret_cast<__nv_bfloat16*>(g.out) + out_row * g.ldo + g.out_col_begin + n_base / 2 + 32 * half, x);
  } else if (qkv_tile) {
    const int pos = g.out_row_begin + m;
#pragma unroll 1
    for (int h = half; h < BN / 64; h += 2) qkv_head_epilogue(g, srow + h * 64, n_base + h * 64, b, pos, valid);
  } else if (EPI == PF_EPI_GATE_RESID && g.epi_staged) {
    constexpr int VEC_PER_ROW = BN / 4, ROWS_PER_IT = 32 / VEC_PER_ROW;
    const int warp = tid >> 5, lane = tid & 31;
    const int c4 = lane % VEC_PER_ROW, rsub = lane / VEC_PER_ROW;
    const float4 gg = __ldg(reinterpret_cast<const float4*>(g.gate + b * g.gate_batch_stride + n_base) + c4);
    float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (g.bias != nullptr) bb = __ldg(reinterpret_cast<const float4*>(g.bias + n_base) + c4);
    float* obase = reinterpret_cast<float*>(g.out) + g.out_col_begin + n_base + 4 * c4;
    const size_t row0 = static_cast<size_t>(b) * g.out_batch_rows + g.out_row_begin + m_base;
#pragma unroll 4
    for (int it = 0; it < 16 / ROWS_PER_IT; ++it) {
      const int rr = warp * 16 + it * ROWS_PER_IT + rsub;
      if (m_base + rr < g.row_count) {
        const float4 a4 = *reinterpret_cast<const float4*>(acc_rows + rr * PITCH + 4 * c4);
        float4* dst = reinterpret_cast<float4*>(obase + (row0 + rr) * g.ldo);
        float4 r4 = *dst;
        r4.x += gg.x * (a4.x + bb.x);
        r4.y += gg.y * (a4.y + bb.y);
        r4.z += gg.z * (a4.z + bb.z);
        r4.w += gg.w * (a4.w + bb.w);
        *dst = r4;
      }
    }
  } else {
#pragma unroll 1
    for (int c = half; c < BN / 32; c += 2) {
      const int n0 = n_base + c * 32;
      float x[32];
      load_bias32(x, srow + c * 32, g.bias ? g.bias + n0 : nullptr);
      if (epi_is_act_bf16(EPI) || EPI == PF_EPI_QKV_GELU) {
#pragma unroll
        for (int i = 0; i < 32; ++i) x[i] = epi_act<EPI>(x[i]);
      }
      if (!valid) continue;
      if (EPI == PF_EPI_STORE_BF16 || epi_is_act_bf16(EPI) || EPI == PF_EPI_QKV_GELU) {
        const int col = (EPI == PF_EPI_QKV_GELU) ? (g.out_col_begin + n0 - g.n_split) : (g.out_col_begin + n0);
        store_bf16x32(reinterpret_cast<__nv_bfloat16*>(g.out) + out_row * g.ldo + col, x);
      } else if (EPI == PF_EPI_STORE_F32) {
        float4* d4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(g.out) + out_row * g.ldo + g.out_col_begin + n0);
#pragma unroll
        for (int i = 0; i < 8; ++i) d4[i] = make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
      } else if (EPI == PF_EPI_GATE_RESID) {
        // each thread read-modify-writes its own row (32 rows x 16 bytes per warp instruction)
        float4* d4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(g.out) + out_row * g.ldo + g.out_col_begin + n0);
        const float4* g4 = reinterpret_cast<const float4*>(g.gate + b * g.gate_batch_stride + n0);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float4 rr = d4[i];
          const float4 gg = __ldg(g4 + i);
          rr.x += gg.x * x[4 * i + 0];
          rr.y += gg.y * x[4 * i + 1];
          rr.z += gg.z * x[4 * i + 2];
          rr.w += gg.w * x[4 * i + 3];
          d4[i] = rr;
        }
      }
    }
  }
}

template <int BN, int EPI>
__global__ void __launch_bounds__(PIPE_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                       const GemmArgs g) {
  using Cfg = PipeCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* acc_tile = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);

  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];

  const int warp = threadIdx.x >> 5;
  const int wgroup = warp >> 2;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], PIPE_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int num_kb = (g.k + BK - 1) / BK;
  const int tiles_per_batch = g.m_tiles * g.n_tiles;
  const int total_tiles = g.batches * tiles_per_batch;

  if (wgroup == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // ===== TMA producer =====
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int b = tile / tiles_per_batch;
        const int r = tile - b * tiles_per_batch;
        const int mt = r / g.n_tiles;
        const int nt = r - mt * g.n_tiles;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          tma_load_3d(sa, &tm_a, &full_bar[stage], kb * BK, g.row_begin + mt * BM, b);
          tma_load_2d(sa + Cfg::A_BYTES, &tm_b, &full_bar[stage], kb * BK, nt * BN);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===== consumers: K loop on the tensor cores, then the epilogue of their own 64 rows =====
    setmaxnreg_inc<232>();
    const int wg = wgroup - 1;
    const int tid = threadIdx.x & 127;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int b = tile / tiles_per_batch;
      const int r = tile - b * tiles_per_batch;
      const int mt = r / g.n_tiles;
      const int nt = r - mt * g.n_tiles;
      pipe_consume_tile<BN>(acc, smem, full_bar, empty_bar, num_kb, wg, stage, phase);
      named_bar_sync(1 + wg, 128);   // the previous tile's epilogue reads of this warpgroup's staging rows are done
      pipe_stage_acc<BN>(acc, acc_tile, wg);
      named_bar_sync(1 + wg, 128);
      epilogue_tile<BN, EPI>(g, acc_tile + wg * 64 * Cfg::ACC_PITCH, tid, b, mt * BM + wg * 64, nt * BN);
    }
  }
}

// ---- 256 x 128 tiles in 2-CTA clusters ----------------------------------------------------------------------------------
// The two CTAs of a cluster take adjacent 256-row tiles (same batch, same 128 columns).  Each producer loads its own A box
// [256 x 64] and half of the W box [64 x 64], multicast into both CTAs, so a stage (32 KB A + 16 KB W) costs each SM 40 KB of
// L2 -> shared traffic for 4.2 MFLOP.  A stage may be refilled only when the consumers of both CTAs are done with it: every
// consumer warp arrives on its own and on the peer's empty barrier (16 arrivals per phase).
constexpr int CBM = 256;
constexpr int CBN = 128;
// The cluster kernel's two operand types.  A stage row is one 128-byte swizzle row of K in both: 64 bf16 or 128 e4m3.
//   bf16: 256-row tiles; each consumer warpgroup owns two 64-row halves (H = 2).
//   e4m3: 128-row tiles; one 64-row half per warpgroup (H = 1), so that the promotion fragments of
//         cluster_consume_tile_fp8 fit in the register file next to the accumulators.
template <bool FP8>
struct ClusterCfg {
  static constexpr int H = FP8 ? 1 : 2;
  static constexpr int BM = 128 * H;
  static constexpr int BK = FP8 ? 128 : 64;
  static constexpr int STAGES = FP8 ? 6 : 4;
  static constexpr int A_BYTES = BM * 128;
  static constexpr int B_BYTES = CBN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;
};
using Cfg16 = ClusterCfg<false>;
using Cfg8 = ClusterCfg<true>;
static_assert(Cfg16::BM == CBM && Cfg16::BK == BK, "bf16 cluster tile");

// acc[h][64 x 128] (+)= rows [128 wg + 64 h, +64) of the stage's A box . W box^T, for one tile's K loop
__device__ __forceinline__ void cluster_consume_tile(float (&acc)[2][64], uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                                     int num_kb, int wg, int& stage, uint32_t& phase) {
  constexpr int C_STAGES = Cfg16::STAGES;
  const int lane = threadIdx.x & 31;
  int prev = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(smem + stage * Cfg16::STAGE_BYTES);
    const uint64_t da0 = make_smem_desc_kmajor_sw128(sa + (2 * wg + 0) * (64 * 128));
    const uint64_t da1 = make_smem_desc_kmajor_sw128(sa + (2 * wg + 1) * (64 * 128));
    const uint64_t db = make_smem_desc_kmajor_sw128(sa + Cfg16::A_BYTES);
    wgmma_reg_fence(acc[0]);
    wgmma_reg_fence(acc[1]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) {
      const uint32_t accum = (kb | kk) != 0 ? 1u : 0u;
      wgmma_ss_n128(acc[0], da0 + 2 * kk, db + 2 * kk, accum);
      wgmma_ss_n128(acc[1], da1 + 2 * kk, db + 2 * kk, accum);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && lane == 0) {
      mbar_arrive_cluster(&empty_bar[prev], 0);
      mbar_arrive_cluster(&empty_bar[prev], 1);
    }
    prev = stage;
    if (++stage == C_STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  wgmma_reg_fence(acc[0]);
  wgmma_reg_fence(acc[1]);
  if (prev >= 0 && lane == 0) {
    mbar_arrive_cluster(&empty_bar[prev], 0);
    mbar_arrive_cluster(&empty_bar[prev], 1);
  }
}

// t[64 x 128] = rows [64 wg, +64) of an e4m3 stage's A box . W box^T over the stage's K = 128 (four k32 steps), committed
// as one wgmma group
__device__ __forceinline__ void fp8_stage_mma(float (&t)[64], uint8_t* smem, int stage, int wg) {
  const uint32_t sa = smem_u32(smem + stage * Cfg8::STAGE_BYTES);
  const uint64_t da = make_smem_desc_kmajor_sw128(sa + wg * (64 * 128));
  const uint64_t db = make_smem_desc_kmajor_sw128(sa + Cfg8::A_BYTES);
  wgmma_reg_fence(t);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < Cfg8::BK / 32; ++kk) wgmma_ss_n128_e4m3(t, da + 2 * kk, db + 2 * kk, kk != 0 ? 1u : 0u);
  wgmma_commit();
}

// acc[0][64 x 128] = rows [64 wg, +64) of the tile, e4m3 operands.  Hopper's fp8 wgmma adds products into its accumulator
// with reduced internal precision (about 14 bits), which over K = 9600 loses about 1e-2 relative.  So each stage (K = 128)
// runs into a fresh fragment t, which is added into the fp32 accumulator with FADD once its group has retired (promotion);
// the sum order depends on K only.  The fragment is read only after wait<0>: reading one while another group of the same
// warpgroup is in flight makes ptxas serialise every wgmma (C7514).  The other consumer warpgroup's wgmmas fill the gap.
__device__ __forceinline__ void cluster_consume_tile_fp8(float (&acc)[1][64], uint8_t* smem, uint64_t* full_bar,
                                                         uint64_t* empty_bar, int num_kb, int wg, int& stage, uint32_t& phase) {
  const int lane = threadIdx.x & 31;
  float t[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[0][i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    fp8_stage_mma(t, smem, stage, wg);
    wgmma_wait<0>();
    wgmma_reg_fence(t);
    if (lane == 0) {
      mbar_arrive_cluster(&empty_bar[stage], 0);
      mbar_arrive_cluster(&empty_bar[stage], 1);
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[0][i] += t[i];
    if (++stage == Cfg8::STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
}

// Epilogue straight from the accumulator fragments (pf_common.cuh wgmma layout): thread (warp w, lane l) of consumer
// warpgroup wg holds, for h < H, half in {0, 1}, tile row 64 (H wg + h) + 16 w + l / 4 + 8 half at columns 8 i + 2 (l % 4)
// + {0, 1}, i = 0..15, in acc[h][4 i + 2 half + {0, 1}].  Unscaled (bf16): same arithmetic per element, in the same order, as
// the staged epilogue of the 128-row kernels: the same bits.  SCALED (e4m3): each accumulator is first multiplied by its
// row's a_scale and then its column's w_scale; what follows is the same arithmetic.
template <int EPI, int H, bool SCALED>
__device__ __forceinline__ void epilogue_frag(const GemmArgs& g, const float (&acc)[H][64], int wg, int b, int m_base, int n_base) {
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int r_thr = wg * 64 * H + w * 16 + (lane >> 2);   // + 64 h + 8 half
  const int c_thr = 2 * (lane & 3);                       // + 8 i
  bool qkv_tile = (EPI == PF_EPI_QKV_ROPE);
  if (EPI == PF_EPI_QKV_GELU) qkv_tile = n_base < g.n_split;
  float sa[2 * H];   // row scales of (h, half)
  if constexpr (SCALED) {
#pragma unroll
    for (int hr = 0; hr < 2 * H; ++hr) {
      const int m = m_base + r_thr + 64 * (hr >> 1) + 8 * (hr & 1);
      sa[hr] = m < g.row_count ? __ldg(g.a_scale + static_cast<size_t>(b) * g.rows_per_batch + g.row_begin + m) : 0.f;
    }
  }
  // the accumulator of (h, half) = hr at column n (n even): dequantised pair (n, n + 1)
  auto value2 = [&](int hr, int idx, int n) -> float2 {
    const float a0 = acc[hr >> 1][idx], a1 = acc[hr >> 1][idx + 1];
    if constexpr (SCALED) {
      const float2 ws = __ldg(reinterpret_cast<const float2*>(g.w_scale + n));
      return make_float2(a0 * sa[hr] * ws.x, a1 * sa[hr] * ws.y);
    } else {
      return make_float2(a0, a1);
    }
  };

  if constexpr (EPI == PF_EPI_GEGLU_BF16) {
    // column group i < 8 is the gate, i + 8 the linear term of the same thread: output column n_base / 2 + 8 i + c_thr
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int n = n_base + 8 * i + c_thr;
      float2 bg = make_float2(0.f, 0.f), bl = make_float2(0.f, 0.f);
      if (g.bias != nullptr) {
        bg = __ldg(reinterpret_cast<const float2*>(g.bias + n));
        bl = __ldg(reinterpret_cast<const float2*>(g.bias + n + 64));
      }
#pragma unroll
      for (int hr = 0; hr < 2 * H; ++hr) {
        const int h = hr >> 1, half = hr & 1;
        const int m = m_base + r_thr + 64 * h + 8 * half;
        const float2 ga = value2(hr, 4 * i + 2 * half, n);
        const float2 la = value2(hr, 4 * (i + 8) + 2 * half, n + 64);
        const float x0 = gelu_tanh_f(ga.x + bg.x) * (la.x + bl.x);
        const float x1 = gelu_tanh_f(ga.y + bg.y) * (la.y + bl.y);
        if (m >= g.row_count) continue;
        const size_t out_row = static_cast<size_t>(b) * g.out_batch_rows + g.out_row_begin + m;
        *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(g.out) + out_row * g.ldo + g.out_col_begin + n_base / 2 + 8 * i +
                                     c_thr) = pack_bf16x2(x0, x1);
      }
    }
  } else if (qkv_tile) {
    const int inner = g.heads * g.head_dim;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {   // the tile's two 64-column heads
      const int n0 = n_base + hh * 64;
      const int section = n0 / inner;
      const int head = (n0 - section * inner) / g.head_dim;
      __nv_bfloat16* base = section == 0 ? g.q_out : (section == 1 ? g.k_out : g.v_out);
      const float* nw = section == 0 ? g.q_norm_w : g.k_norm_w;
#pragma unroll
      for (int hr = 0; hr < 2 * H; ++hr) {
        const int h = hr >> 1, half = hr & 1;
        const int m = m_base + r_thr + 64 * h + 8 * half;
        const bool valid = m < g.row_count;
        const int pos = g.out_row_begin + m;
        float x[16];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float2 bb = make_float2(0.f, 0.f);
          if (g.bias != nullptr) bb = __ldg(reinterpret_cast<const float2*>(g.bias + n0 + 8 * j + c_thr));
          const float2 a = value2(hr, 4 * (8 * hh + j) + 2 * half, n0 + 8 * j + c_thr);
          x[2 * j + 0] = a.x + bb.x;
          x[2 * j + 1] = a.y + bb.y;
        }
        if (section < 2) {   // RMSNorm over the head (N:66-79), then RoPE (B:34-39)
          // The staged epilogue's sum order: chain c (0..3) runs over columns 4 k + c, k ascending, and the head's sum is
          // (s0 + s1) + (s2 + s3).  Columns 4 k + c alternate between the threads t and t ^ 2 of the row (8 j + 2 t + e
          // = 4 (2 j + t / 2) + 2 (t % 2) + e), so each thread fetches its partner's values and runs chains 2 (t % 2) + e.
          const bool lo_first = (lane & 2) == 0;
          float s_e[2] = {0.f, 0.f};
#pragma unroll
          for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float own = x[2 * j + e], other = __shfl_xor_sync(0xffffffffu, own, 2);
              const float first = lo_first ? own : other, second = lo_first ? other : own;
              s_e[e] = fmaf(first, first, s_e[e]);
              s_e[e] = fmaf(second, second, s_e[e]);
            }
          }
          const float pair = s_e[0] + s_e[1];                           // s0 + s1 (t even) or s2 + s3 (t odd)
          const float ss = pair + __shfl_xor_sync(0xffffffffu, pair, 1);   // fp32 add commutes: same bits in all four
          const float r = rsqrtf(ss * (1.0f / 64.0f) + g.norm_eps);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 wn = __ldg(reinterpret_cast<const float2*>(nw + 8 * j + c_thr));
            x[2 * j + 0] *= r * wn.x;
            x[2 * j + 1] *= r * wn.y;
          }
          if (g.rope != nullptr && valid) {
            const float* rp = g.rope + static_cast<size_t>(pos) * 64 + c_thr;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float2 cs = __ldg(reinterpret_cast<const float2*>(rp + 8 * j));   // (cos, sin) of pair 4 j + l % 4
              const float a0 = x[2 * j + 0], a1 = x[2 * j + 1];
              x[2 * j + 0] = cs.x * a0 - cs.y * a1;
              x[2 * j + 1] = cs.y * a0 + cs.x * a1;
            }
          }
        }
        if (valid) {
          __nv_bfloat16* dst;
          if (g.peer_count > 1) {
            const int pr = head / g.peer_heads, hl = head - pr * g.peer_heads;
            dst = g.peer_qkv[pr] + ((static_cast<size_t>(section) * g.peer_heads + hl) * g.peer_seq + g.peer_row0 + pos) * 64;
          } else {
            dst = base + ((static_cast<size_t>(b) * g.heads + head) * g.seq_len + pos) * 64;
          }
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<uint32_t*>(dst + 8 * j + c_thr) = pack_bf16x2(x[2 * j + 0], x[2 * j + 1]);
        }
      }
    }
  } else if (EPI == PF_EPI_GATE_RESID) {
    // fp32 read-modify-write of the residual: a row's four threads cover 32 contiguous bytes per column group; all 16 loads
    // of a row are issued before its stores
    const float* gate = g.gate + b * g.gate_batch_stride + n_base + c_thr;
    float* obase = reinterpret_cast<float*>(g.out) + g.out_col_begin + n_base + c_thr;
#pragma unroll
    for (int hr = 0; hr < 2 * H; ++hr) {
      const int h = hr >> 1, half = hr & 1;
      const int m = m_base + r_thr + 64 * h + 8 * half;
      if (m >= g.row_count) continue;
      float2* dst = reinterpret_cast<float2*>(obase + (static_cast<size_t>(b) * g.out_batch_rows + g.out_row_begin + m) * g.ldo);
      float2 rr[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) rr[i] = dst[4 * i];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float2 bb = make_float2(0.f, 0.f);
        if (g.bias != nullptr) bb = __ldg(reinterpret_cast<const float2*>(g.bias + n_base + 8 * i + c_thr));
        const float2 gg = __ldg(reinterpret_cast<const float2*>(gate + 8 * i));
        const float2 a = value2(hr, 4 * i + 2 * half, n_base + 8 * i + c_thr);
        const float x0 = a.x + bb.x;
        const float x1 = a.y + bb.y;
        rr[i].x += gg.x * x0;
        rr[i].y += gg.y * x1;
        dst[4 * i] = rr[i];
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int n = n_base + 8 * i + c_thr;
      float2 bb = make_float2(0.f, 0.f);
      if (g.bias != nullptr) bb = __ldg(reinterpret_cast<const float2*>(g.bias + n));
#pragma unroll
      for (int hr = 0; hr < 2 * H; ++hr) {
        const int h = hr >> 1, half = hr & 1;
        const int m = m_base + r_thr + 64 * h + 8 * half;
        const float2 a = value2(hr, 4 * i + 2 * half, n);
        float x0 = a.x + bb.x;
        float x1 = a.y + bb.y;
        if (epi_is_act_bf16(EPI) || EPI == PF_EPI_QKV_GELU) {
          x0 = epi_act<EPI>(x0);
          x1 = epi_act<EPI>(x1);
        }
        if (m >= g.row_count) continue;
        const size_t out_row = static_cast<size_t>(b) * g.out_batch_rows + g.out_row_begin + m;
        if (EPI == PF_EPI_STORE_F32) {
          *reinterpret_cast<float2*>(reinterpret_cast<float*>(g.out) + out_row * g.ldo + g.out_col_begin + n) = make_float2(x0, x1);
        } else {
          const int col = (EPI == PF_EPI_QKV_GELU) ? (g.out_col_begin + n - g.n_split) : (g.out_col_begin + n);
          *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(g.out) + out_row * g.ldo + col) = pack_bf16x2(x0, x1);
        }
      }
    }
  }
}

template <int EPI, bool FP8>
__global__ void __launch_bounds__(PIPE_THREADS, 1)
gemm_cluster_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b, const GemmArgs g) {
  using Cfg = ClusterCfg<FP8>;
  constexpr int C_STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  __shared__ __align__(8) uint64_t full_bar[C_STAGES];
  __shared__ __align__(8) uint64_t empty_bar[C_STAGES];

  const int warp = threadIdx.x >> 5;
  const int wgroup = warp >> 2;
  const uint32_t rank = cluster_ctarank();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
    for (int i = 0; i < C_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2 * PIPE_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  // the peer's barriers are initialised before anything arrives on them or multicasts into its shared memory
  cluster_arrive();
  cluster_wait();

  // Static schedule over tile pairs: both CTAs of a cluster walk the same pairs.  m_tiles is even-padded per batch; the
  // partner of an odd last tile loads rows past row_count (zero-filled or masked) and stores nothing.
  const int num_kb = (g.k + Cfg::BK - 1) / Cfg::BK;
  const int m_pairs = (g.m_tiles + 1) >> 1;
  const int pairs_per_batch = m_pairs * g.n_tiles;
  const int total_pairs = g.batches * pairs_per_batch;
  const int cluster = blockIdx.x >> 1, clusters = gridDim.x >> 1;

  if (wgroup == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // ===== TMA producer =====
      int stage = 0;
      uint32_t phase = 0;
      for (int p = cluster; p < total_pairs; p += clusters) {
        const int b = p / pairs_per_batch;
        const int r = p - b * pairs_per_batch;
        const int mt = 2 * (r / g.n_tiles) + static_cast<int>(rank);
        const int nt = r % g.n_tiles;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          tma_load_3d(sa, &tm_a, &full_bar[stage], kb * Cfg::BK, g.row_begin + mt * Cfg::BM, b);
          tma_load_2d_multicast(sa + Cfg::A_BYTES + rank * (Cfg::B_BYTES / 2), &tm_b, &full_bar[stage], kb * Cfg::BK,
                                nt * CBN + rank * (CBN / 2), 0x3);
          if (++stage == C_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ===== consumers: each warpgroup owns 64 H rows of the tile =====
    setmaxnreg_inc<232>();
    const int wg = wgroup - 1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[Cfg::H][64];
    for (int p = cluster; p < total_pairs; p += clusters) {
      const int b = p / pairs_per_batch;
      const int r = p - b * pairs_per_batch;
      const int mt = 2 * (r / g.n_tiles) + static_cast<int>(rank);
      const int nt = r % g.n_tiles;
      if constexpr (FP8) cluster_consume_tile_fp8(acc, smem, full_bar, empty_bar, num_kb, wg, stage, phase);
      else cluster_consume_tile(acc, smem, full_bar, empty_bar, num_kb, wg, stage, phase);
      epilogue_frag<EPI, Cfg::H, FP8>(g, acc, wg, b, mt * Cfg::BM, nt * CBN);
    }
  }
  // no CTA exits while its peer may still arrive on its barriers
  cluster_arrive();
  cluster_wait();
}

template <int BN, int EPI>
static int launch_gemm(const CUtensorMap& tm_a, const CUtensorMap& tm_b, const GemmArgs& g, cudaStream_t stream) {
  using Cfg = PipeCfg<BN>;
  auto kern = gemm_bf16_wgmma_kernel<BN, EPI>;
  if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), Cfg::SMEM_BYTES, "gemm")) return rc;
  const int total = g.batches * g.m_tiles * g.n_tiles;
  int grid = num_sms();
  if (grid <= 0) grid = 132;
  if (total < grid) grid = total;
  kern<<<grid, PIPE_THREADS, Cfg::SMEM_BYTES, stream>>>(tm_a, tm_b, g);
  return check_launch("pf_gemm_bf16");
}

// Clusters of the cluster kernel that fit on the device at once (SMs pair up within a GPC, so this can be below
// num_sms() / 2); queried once, before any CUDA-graph capture, by warmup_gemm.  Both operand types take one CTA per SM and
// the same shared memory.
static_assert(Cfg8::SMEM_BYTES == Cfg16::SMEM_BYTES, "one cluster occupancy for both operand types");
static int g_cluster_slots = 0;

static int cluster_slots() {
  if (g_cluster_slots > 0) return g_cluster_slots;
  auto kern = gemm_cluster_kernel<PF_EPI_STORE_BF16, false>;
  if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), Cfg16::SMEM_BYTES, "gemm cluster")) return rc;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.gridDim = dim3(2, 1, 1);
  cfg.blockDim = dim3(PIPE_THREADS, 1, 1);
  cfg.dynamicSmemBytes = Cfg16::SMEM_BYTES;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess || n <= 0) {
    (void)cudaGetLastError();
    n = num_sms() > 0 ? num_sms() / 2 : 66;
  }
  g_cluster_slots = n;
  return n;
}

template <int EPI, bool FP8 = false>
static int launch_cluster(const CUtensorMap& tm_a, const CUtensorMap& tm_b, const GemmArgs& g, cudaStream_t stream) {
  auto kern = gemm_cluster_kernel<EPI, FP8>;
  constexpr int smem_bytes = ClusterCfg<FP8>::SMEM_BYTES;
  if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), smem_bytes, "gemm cluster")) return rc;
  const int slots = cluster_slots();
  if (slots < 0) return slots;
  const int pairs = g.batches * ((g.m_tiles + 1) / 2) * g.n_tiles;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.gridDim = dim3(2 * (pairs < slots ? pairs : slots), 1, 1);
  cfg.blockDim = dim3(PIPE_THREADS, 1, 1);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  (void)cudaLaunchKernelEx(&cfg, kern, tm_a, tm_b, g);
  return check_launch(FP8 ? "pf_gemm_fp8" : "pf_gemm_bf16");
}

// tile 0 = 256 x 128 in 2-CTA clusters, else the 128-row kernel with BLOCK_N = tile
template <int EPI>
static int dispatch_tile(int tile, const CUtensorMap& tm_a, const CUtensorMap& tm_b, const GemmArgs& g, cudaStream_t stream) {
  switch (tile) {
    case 0: return launch_cluster<EPI>(tm_a, tm_b, g, stream);
    case 128: return launch_gemm<128, EPI>(tm_a, tm_b, g, stream);
    case 64:
      if constexpr (EPI != PF_EPI_GEGLU_BF16) return launch_gemm<64, EPI>(tm_a, tm_b, g, stream);
      break;
  }
  set_error("unsupported GEMM tile %d", tile);
  return -1;
}

// the text-encoder epilogues (> QKV_GELU) have no fp8 instantiation, and GEGLU none on the 128 x 64 kernel
template <int EPI>
static int warm_epi() {
  int rc = ensure_dyn_smem(reinterpret_cast<const void*>(gemm_cluster_kernel<EPI, false>), Cfg16::SMEM_BYTES, "gemm cluster");
  if constexpr (EPI <= PF_EPI_QKV_GELU)
    if (!rc) rc = ensure_dyn_smem(reinterpret_cast<const void*>(gemm_cluster_kernel<EPI, true>), Cfg8::SMEM_BYTES, "gemm cluster fp8");
  if (!rc) rc = ensure_dyn_smem(reinterpret_cast<const void*>(gemm_bf16_wgmma_kernel<128, EPI>), PipeCfg<128>::SMEM_BYTES, "gemm<128>");
  if constexpr (EPI != PF_EPI_GEGLU_BF16)
    if (!rc) rc = ensure_dyn_smem(reinterpret_cast<const void*>(gemm_bf16_wgmma_kernel<64, EPI>), PipeCfg<64>::SMEM_BYTES, "gemm<64>");
  return rc;
}
// load every instantiation and set its dynamic-smem attribute on the current device (so nothing initialises inside a
// CUDA-graph capture)
int warmup_gemm() {
  int rc = warm_epi<PF_EPI_STORE_BF16>();
  if (!rc) rc = warm_epi<PF_EPI_GELU_BF16>();
  if (!rc) rc = warm_epi<PF_EPI_STORE_F32>();
  if (!rc) rc = warm_epi<PF_EPI_GATE_RESID>();
  if (!rc) rc = warm_epi<PF_EPI_QKV_ROPE>();
  if (!rc) rc = warm_epi<PF_EPI_QKV_GELU>();
  if (!rc) rc = warm_epi<PF_EPI_GEGLU_BF16>();
  if (!rc) rc = warm_epi<PF_EPI_QUICK_GELU_BF16>();
  if (!rc) rc = warm_epi<PF_EPI_GELU_ERF_BF16>();
  if (!rc) rc = cluster_slots() > 0 ? 0 : -1;
  return rc;
}

// Validation shared by both entries (everything except the operand format), then the kernel arguments from the descriptor.
// `fn` names the entry in the messages; `k_align` = elements per 16 bytes of A / W (TMA row strides).
static int gemm_args_from_desc(const pf_gemm_desc* d, const char* fn, int k_align, GemmArgs& g) {
  PF_REQUIRE(d->a && d->w, "%s: null operand", fn);
  PF_REQUIRE(d->k > 0 && d->k % k_align == 0, "%s: k=%d must be a positive multiple of %d", fn, d->k, k_align);
  PF_REQUIRE(d->lda % k_align == 0 && d->lda >= d->k, "%s: lda=%lld must be >= k and a multiple of %d", fn, (long long)d->lda,
             k_align);
  PF_REQUIRE(d->batches > 0 && d->rows_per_batch > 0 && d->row_count > 0 && d->row_begin >= 0 &&
                 d->row_begin + d->row_count <= d->rows_per_batch,
             "%s: bad row range (batches %d rows %d begin %d count %d)", fn, d->batches, d->rows_per_batch,
             d->row_begin, d->row_count);
  PF_REQUIRE((reinterpret_cast<uintptr_t>(d->a) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->w) & 15) == 0,
             "%s: operands must be 16-byte aligned", fn);
  const int epi = d->epilogue;
  PF_REQUIRE(epi >= 0 && epi <= PF_EPI_GELU_ERF_BF16, "%s: unknown epilogue %d", fn, epi);
  if (epi == PF_EPI_GEGLU_BF16)
    PF_REQUIRE(d->n % 128 == 0 && d->kernel_variant != 2,
               "%s: GEGLU needs n %% 128 == 0 (n=%d) and 128-wide tiles (kernel_variant %d)", fn, d->n, d->kernel_variant);

  // The QKV epilogues work per 64-column head, so any multiple of 64 is head-aligned.
  const bool qkv = (epi == PF_EPI_QKV_ROPE || epi == PF_EPI_QKV_GELU);
  if (qkv) {
    PF_REQUIRE(d->head_dim == 64, "%s: QKV epilogue supports head_dim 64 only (got %d)", fn, d->head_dim);
    const int inner = d->heads * d->head_dim;
    const int nq = 3 * inner;
    PF_REQUIRE(d->q_out && d->k_out && d->v_out && d->q_norm_w && d->k_norm_w, "%s: QKV epilogue needs q/k/v outputs and norm weights", fn);
    PF_REQUIRE(d->out_row_begin + d->row_count <= d->seq_len, "%s: QKV rows exceed seq_len", fn);
    if (epi == PF_EPI_QKV_ROPE) {
      PF_REQUIRE(d->n == nq, "%s: QKV_ROPE needs n == 3*heads*head_dim", fn);
    } else {
      PF_REQUIRE(d->n_split == nq && d->n > nq && d->out != nullptr, "%s: QKV_GELU needs n_split == 3*heads*head_dim < n and out", fn);
      PF_REQUIRE(nq % 64 == 0, "%s: n_split must be a multiple of 64", fn);
    }
  } else {
    PF_REQUIRE(d->out != nullptr, "%s: null output", fn);
    if (epi == PF_EPI_GATE_RESID) PF_REQUIRE(d->gate != nullptr, "%s: GATE_RESID needs gate", fn);
    const int esz = (epi == PF_EPI_STORE_F32 || epi == PF_EPI_GATE_RESID) ? 4 : 2;
    PF_REQUIRE((d->ldo * esz) % 16 == 0 && (d->out_col_begin * esz) % 16 == 0 &&
                   (reinterpret_cast<uintptr_t>(d->out) & 15) == 0,
               "%s: output must be 16-byte aligned (ldo %lld col %d)", fn, (long long)d->ldo, d->out_col_begin);
  }
  PF_REQUIRE(d->n % 64 == 0, "%s: n=%d must be a multiple of 64", fn, d->n);

  g = GemmArgs{};
  g.batches = d->batches;
  g.row_begin = d->row_begin;
  g.row_count = d->row_count;
  g.n = d->n;
  g.k = d->k;
  g.bias = d->bias;
  g.out = d->out;
  g.ldo = d->ldo;
  g.out_batch_rows = d->out_batch_rows;
  g.out_row_begin = d->out_row_begin;
  g.out_col_begin = d->out_col_begin;
  g.gate = d->gate;
  g.gate_batch_stride = d->gate_batch_stride;
  g.q_out = static_cast<__nv_bfloat16*>(d->q_out);
  g.k_out = static_cast<__nv_bfloat16*>(d->k_out);
  g.v_out = static_cast<__nv_bfloat16*>(d->v_out);
  g.rope = d->rope;
  g.q_norm_w = d->q_norm_w;
  g.k_norm_w = d->k_norm_w;
  g.norm_eps = d->norm_eps;
  g.heads = d->heads;
  g.head_dim = d->head_dim;
  g.seq_len = d->seq_len;
  g.n_split = d->n_split;
  g.epi_staged = get_option(PF_OPT_GEMM_STAGED_RESID);
  g.peer_count = d->peer_count;
  g.peer_heads = d->peer_heads;
  g.peer_seq = d->peer_seq;
  g.peer_row0 = d->peer_row0;
  g.rows_per_batch = d->rows_per_batch;
  for (int i = 0; i < PF_MAX_PEERS; ++i) g.peer_qkv[i] = static_cast<__nv_bfloat16*>(d->peer_qkv[i]);
  if (d->peer_count > 1) {
    PF_REQUIRE(epi == PF_EPI_QKV_ROPE && d->batches == 1, "%s: peer stores need the QKV_ROPE epilogue and batches == 1", fn);
    PF_REQUIRE(d->peer_count <= PF_MAX_PEERS && d->peer_heads > 0 && d->peer_heads * d->peer_count >= d->heads &&
                   d->peer_row0 >= 0 && d->peer_row0 + d->out_row_begin + d->row_count <= d->peer_seq,
               "%s: bad peer layout (count %d heads/rank %d seq %d row0 %d)", fn, d->peer_count, d->peer_heads, d->peer_seq, d->peer_row0);
    for (int i = 0; i < d->peer_count; ++i) {
      PF_REQUIRE(d->peer_qkv[i] != nullptr, "%s: peer_qkv[%d] is null", fn, i);
      // the staged epilogue stores 16-byte vectors
      PF_REQUIRE((reinterpret_cast<uintptr_t>(d->peer_qkv[i]) & 15) == 0, "%s: peer_qkv[%d] must be 16-byte aligned", fn, i);
    }
  }
  return 0;
}

}  // namespace pf

extern "C" int pf_gemm_bf16(const pf_gemm_desc* d, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(d != nullptr, "pf_gemm_bf16: null descriptor");
  GemmArgs g;
  if (int rc = gemm_args_from_desc(d, "pf_gemm_bf16", 8, g)) return rc;
  const int epi = d->epilogue;
  // Column tiling: 128-wide tiles when they divide n, else 64-wide.
  // QKV_GELU: tiles must not straddle the q|k|v / mlp boundary (different epilogue per tile)
  int bn = (d->n % 128 == 0 && (epi != PF_EPI_QKV_GELU || d->n_split % 128 == 0)) ? 128 : 64;

  // Kernels: tile 0 = 256 x 128 in 2-CTA clusters (needs 128 | n), 128 = 128 x 128, 64 = 128 x 64.  All three run the same
  // wgmma k16 steps in the same order per output element and the same epilogue arithmetic: same bits whichever runs.
  // kernel_variant 1 pins the 256 x 128 cluster kernel, 2 the 128 x 64 kernel.
  PF_REQUIRE(d->kernel_variant >= 0 && d->kernel_variant <= 2, "pf_gemm_bf16: bad kernel_variant %d", d->kernel_variant);
  PF_REQUIRE(d->kernel_variant != 1 || bn == 128, "pf_gemm_bf16: kernel_variant 1 (128-wide tiles) needs n %% 128 == 0");
  int tile = bn == 128 ? 0 : 64;
  if (d->kernel_variant == 2) tile = 64;
  // Wave quantisation: with few rows (the 128-row text ranges, a sequence-parallel rank's chunk) the big tiles leave most of
  // the last (or only) wave of the persistent grid idle.  Take the kernel with the least waves x tile area / relative rate.
  if (tile == 0 && d->kernel_variant == 0 && get_option(PF_OPT_GEMM_WAVE_TILING)) {
    int sms = num_sms();
    if (sms <= 0) sms = 132;
    const int slots = cluster_slots();
    const long long mt128 = (d->row_count + BM - 1) / BM, mt256 = (d->row_count + CBM - 1) / CBM;
    const long long waves0 = (d->batches * ((mt256 + 1) / 2) * (d->n / 128) + slots - 1) / (slots > 0 ? slots : 66);
    const long long waves128 = (d->batches * mt128 * (d->n / 128) + sms - 1) / sms;
    const long long waves64 = (d->batches * mt128 * (d->n / 64) + sms - 1) / sms;
    const double cost0 = waves0 * 2.0 / GEMM_RATE_CLUSTER, cost128 = waves128 * 1.0 / GEMM_RATE_128,
                 cost64 = waves64 * 0.5 / GEMM_RATE_64;
    const bool allow64 = epi != PF_EPI_GEGLU_BF16;   // GEGLU pairs columns 64 apart inside a 128-wide tile
    if (cost128 < cost0 && (cost128 <= cost64 || !allow64)) tile = 128;
    else if (allow64 && cost64 < cost0) tile = 64;
  }
  if (tile != 0) bn = tile;
  const int tile_rows = tile == 0 ? CBM : BM;
  g.m_tiles = (d->row_count + tile_rows - 1) / tile_rows;
  CUtensorMap tm_a;
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(d->k), static_cast<uint64_t>(d->rows_per_batch),
                              static_cast<uint64_t>(d->batches)};
    const uint64_t strides[2] = {static_cast<uint64_t>(d->lda) * 2,
                                 static_cast<uint64_t>(d->lda) * 2 * static_cast<uint64_t>(d->rows_per_batch)};
    const uint32_t box[3] = {BK, static_cast<uint32_t>(tile_rows), 1};
    int rc = encode_tensor_map(&tm_a, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, d->a, dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }

  CUtensorMap tm_b;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(d->k), static_cast<uint64_t>(d->n)};
    const uint64_t strides[1] = {static_cast<uint64_t>(d->k) * 2};
    const uint32_t box[2] = {BK, static_cast<uint32_t>(tile == 0 ? CBN / 2 : bn)};   // cluster: each CTA loads half
    int rc = encode_tensor_map(&tm_b, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, d->w, dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  g.n_tiles = d->n / bn;
  switch (epi) {
    case PF_EPI_STORE_BF16: return dispatch_tile<PF_EPI_STORE_BF16>(tile, tm_a, tm_b, g, stream);
    case PF_EPI_GELU_BF16: return dispatch_tile<PF_EPI_GELU_BF16>(tile, tm_a, tm_b, g, stream);
    case PF_EPI_STORE_F32: return dispatch_tile<PF_EPI_STORE_F32>(tile, tm_a, tm_b, g, stream);
    case PF_EPI_GATE_RESID: return dispatch_tile<PF_EPI_GATE_RESID>(tile, tm_a, tm_b, g, stream);
    case PF_EPI_QKV_ROPE: return dispatch_tile<PF_EPI_QKV_ROPE>(tile, tm_a, tm_b, g, stream);
    case PF_EPI_QKV_GELU: return dispatch_tile<PF_EPI_QKV_GELU>(tile, tm_a, tm_b, g, stream);
    case PF_EPI_GEGLU_BF16: return dispatch_tile<PF_EPI_GEGLU_BF16>(tile, tm_a, tm_b, g, stream);
    case PF_EPI_QUICK_GELU_BF16: return dispatch_tile<PF_EPI_QUICK_GELU_BF16>(tile, tm_a, tm_b, g, stream);
    case PF_EPI_GELU_ERF_BF16: return dispatch_tile<PF_EPI_GELU_ERF_BF16>(tile, tm_a, tm_b, g, stream);
  }
  return -1;
}

extern "C" int pf_gemm_fp8(const pf_gemm_desc* d, const float* a_row_scale, const float* w_col_scale, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(d != nullptr, "pf_gemm_fp8: null descriptor");
  PF_REQUIRE(a_row_scale != nullptr && w_col_scale != nullptr, "pf_gemm_fp8: null scale (a_row_scale and w_col_scale are required)");
  PF_REQUIRE(d->peer_count <= 0, "pf_gemm_fp8: sequence-parallel peer stores (peer_count %d) are bf16 only", d->peer_count);
  PF_REQUIRE(d->kernel_variant == 0, "pf_gemm_fp8: kernel_variant %d: there is one fp8 kernel (0)", d->kernel_variant);
  PF_REQUIRE(d->n % 128 == 0, "pf_gemm_fp8: n=%d must be a multiple of 128", d->n);
  PF_REQUIRE(d->epilogue != PF_EPI_QKV_GELU || d->n_split % 128 == 0, "pf_gemm_fp8: QKV_GELU needs n_split %% 128 == 0");
  PF_REQUIRE(d->epilogue <= PF_EPI_QKV_GELU, "pf_gemm_fp8: epilogue %d is bf16 only (pf_gemm_bf16)", d->epilogue);
  GemmArgs g;
  if (int rc = gemm_args_from_desc(d, "pf_gemm_fp8", 16, g)) return rc;
  g.a_scale = a_row_scale;
  g.w_scale = w_col_scale;
  g.m_tiles = (d->row_count + Cfg8::BM - 1) / Cfg8::BM;
  g.n_tiles = d->n / CBN;
  CUtensorMap tm_a, tm_b;
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(d->k), static_cast<uint64_t>(d->rows_per_batch),
                              static_cast<uint64_t>(d->batches)};
    const uint64_t strides[2] = {static_cast<uint64_t>(d->lda),
                                 static_cast<uint64_t>(d->lda) * static_cast<uint64_t>(d->rows_per_batch)};
    const uint32_t box[3] = {Cfg8::BK, Cfg8::BM, 1};
    if (int rc = encode_tensor_map(&tm_a, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, d->a, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return rc;
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(d->k), static_cast<uint64_t>(d->n)};
    const uint64_t strides[1] = {static_cast<uint64_t>(d->k)};
    const uint32_t box[2] = {Cfg8::BK, CBN / 2};   // each CTA of the cluster loads half of the W box
    if (int rc = encode_tensor_map(&tm_b, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, d->w, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return rc;
  }
  switch (d->epilogue) {
    case PF_EPI_STORE_BF16: return launch_cluster<PF_EPI_STORE_BF16, true>(tm_a, tm_b, g, stream);
    case PF_EPI_GELU_BF16: return launch_cluster<PF_EPI_GELU_BF16, true>(tm_a, tm_b, g, stream);
    case PF_EPI_STORE_F32: return launch_cluster<PF_EPI_STORE_F32, true>(tm_a, tm_b, g, stream);
    case PF_EPI_GATE_RESID: return launch_cluster<PF_EPI_GATE_RESID, true>(tm_a, tm_b, g, stream);
    case PF_EPI_QKV_ROPE: return launch_cluster<PF_EPI_QKV_ROPE, true>(tm_a, tm_b, g, stream);
    case PF_EPI_QKV_GELU: return launch_cluster<PF_EPI_QKV_GELU, true>(tm_a, tm_b, g, stream);
  }
  return -1;
}
