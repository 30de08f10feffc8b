// pf_text.cu — the text encoders' own kernels (T5 v1.1 encoder, CLIP text transformer): short-sequence attention with an
// additive per-head bias and a key padding mask, the T5 RMSNorm and the token (+ position) embedding lookup.
// The GEMMs of both encoders run on pf_gemm_bf16 (pf_gemm.cu), CLIP's LayerNorms on pf_ln_modulate.
// Op sites (transformers 5.5) are cited in include/pf_b200.h next to each entry point.
//
// pf_attn_fwd_text: one CTA = one (batch, head, 128-row q tile); 384 threads, the house structure of pf_attn.cu:
//   warpgroup 0 (one lane)  TMA producer: the Q tile, then every K tile, then every V tile of the head (seq <= 256, so at
//                           most two 128-row tiles each), each group behind its own mbarrier; nothing is refilled.
//   warpgroups 1, 2         64 q rows each: S = Q.K^T over the whole key range lands in registers (NKV x 64 floats per
//                           thread), scale, bias, key mask and causal mask are applied on the accumulator fragments, the
//                           row softmax is exact (one max, one sum: no online rescaling), P is re-packed in registers as the
//                           bf16 A operand and O = P.V is a wgmma with A from registers and V from smem MN-major.
// Q, K and V are read through one 3-D tensor map over the packed QKV GEMM output [batch][seq][ld_qkv]: q of head h at
// column 64 h, k at 64 (heads + h), v at 64 (2 heads + h).  Rows past seq are zero-filled by TMA and masked as keys.
#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

constexpr int TXT_BM = 128;
constexpr int TXT_BN = 128;
constexpr int TXT_HD = 64;
constexpr int TXT_MAX_SEQ = 256;
constexpr int TXT_THREADS = 384;
constexpr int TXT_TILE_BYTES = TXT_BN * TXT_HD * 2;                       // 16 KB
constexpr int TXT_SMEM_BYTES = (1 + 2 * (TXT_MAX_SEQ / TXT_BN)) * TXT_TILE_BYTES + 1024;

struct TextAttnArgs {
  __nv_bfloat16* out;
  long long ldo;
  int heads, seq;
  float scale;
  const float* bias;        // [heads, 2 seq - 1] or null
  const int* key_mask;      // [batch, seq] or null
  int causal;
};

template <int NKV>
__global__ void __launch_bounds__(TXT_THREADS, 1)
attn_text_kernel(const __grid_constant__ CUtensorMap tm_qkv, const TextAttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_k = smem + TXT_TILE_BYTES;
  uint8_t* smem_v = smem_k + NKV * TXT_TILE_BYTES;
  __shared__ __align__(8) uint64_t bar_qk, bar_v;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wgroup = warp >> 2;
  const int qt = blockIdx.x;
  const int h = blockIdx.y;
  const int b = blockIdx.z;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_qkv);
    mbar_init(&bar_qk, 1);
    mbar_init(&bar_v, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (wgroup == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      mbar_arrive_expect_tx(&bar_qk, (1 + NKV) * TXT_TILE_BYTES);
      tma_load_3d(smem_q, &tm_qkv, &bar_qk, h * TXT_HD, qt * TXT_BM, b);
#pragma unroll
      for (int j = 0; j < NKV; ++j)
        tma_load_3d(smem_k + j * TXT_TILE_BYTES, &tm_qkv, &bar_qk, (a.heads + h) * TXT_HD, j * TXT_BN, b);
      mbar_arrive_expect_tx(&bar_v, NKV * TXT_TILE_BYTES);
#pragma unroll
      for (int j = 0; j < NKV; ++j)
        tma_load_3d(smem_v + j * TXT_TILE_BYTES, &tm_qkv, &bar_v, (2 * a.heads + h) * TXT_HD, j * TXT_BN, b);
    }
    return;
  }

  // ===== consumers: thread (warp w of the warpgroup, g = lane / 4, t = lane % 4) holds rows 16 w + g and 16 w + g + 8 of its
  // warpgroup's 64 q rows, columns 8 i + 2 t + {0, 1} of every 8-column group i of each 128-wide key tile =====
  setmaxnreg_inc<232>();
  const int wg = wgroup - 1;
  const int t4 = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  float s[NKV][64];

  mbar_wait(&bar_qk, 0);
  {
    const uint64_t dq = make_smem_desc_kmajor_sw128(smem_u32(smem_q) + wg * (64 * 128));
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < NKV; ++j) {
      const uint64_t dk = make_smem_desc_kmajor_sw128(smem_u32(smem_k + j * TXT_TILE_BYTES));
#pragma unroll
      for (int kk = 0; kk < TXT_HD / 16; ++kk) wgmma_ss_n128(s[j], dq + 2 * kk, dk + 2 * kk, kk != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < NKV; ++j) wgmma_reg_fence(s[j]);
  }

  // ---- scores: scale * q.k + bias[h, kv - q + seq - 1]; masked keys (padding, kv >= seq, causal kv > q) -> -inf
  const int* km = a.key_mask ? a.key_mask + static_cast<size_t>(b) * a.seq : nullptr;
  const float* bias_h = a.bias ? a.bias + static_cast<size_t>(h) * (2 * a.seq - 1) : nullptr;
  int qpos[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) qpos[r] = qt * TXT_BM + row0 + 8 * r;
#pragma unroll
  for (int j = 0; j < NKV; ++j) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int kv = j * TXT_BN + 8 * i + 2 * t4 + e;
        const bool key_ok = kv < a.seq && (km == nullptr || __ldg(km + kv) != 0);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float& x = s[j][4 * i + 2 * r + e];
          // a q row past seq is never stored: clamp its bias index inside the table
          const int q = qpos[r] < a.seq ? qpos[r] : a.seq - 1;
          const bool ok = key_ok && !(a.causal && kv > q);
          float v = x * a.scale;
          if (bias_h != nullptr && kv < a.seq) v += __ldg(bias_h + (kv - q + a.seq - 1));
          x = ok ? v : -INFINITY;
        }
      }
    }
  }

  // ---- exact row softmax on the fragments (a row's 4 threads reduce with two shuffles)
  constexpr float LOG2E = 1.4426950408889634f;
  float inv_l[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < NKV; ++j)
#pragma unroll
      for (int i = 0; i < 16; ++i) mx = fmaxf(mx, fmaxf(s[j][4 * i + 2 * r], s[j][4 * i + 2 * r + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_ref = (mx == -INFINITY) ? 0.f : mx * LOG2E;   // a row with no key gives zeros
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < NKV; ++j)
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = ex2_approx_f(fmaf(s[j][4 * i + 2 * r + e], LOG2E, -m_ref));
          s[j][4 * i + 2 * r + e] = p;
          sum += p;
        }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    inv_l[r] = sum > 0.f ? 1.f / sum : 0.f;
  }

  // ---- O = P.V: the S fragment of columns [16 kk, 16 kk + 16) of key tile j is the A fragment of k step 8 j + kk
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  uint32_t pa[NKV][TXT_BN / 16][4];
#pragma unroll
  for (int j = 0; j < NKV; ++j)
#pragma unroll
    for (int kk = 0; kk < TXT_BN / 16; ++kk) {
      pa[j][kk][0] = pack_bf16x2(s[j][8 * kk + 0], s[j][8 * kk + 1]);
      pa[j][kk][1] = pack_bf16x2(s[j][8 * kk + 2], s[j][8 * kk + 3]);
      pa[j][kk][2] = pack_bf16x2(s[j][8 * kk + 4], s[j][8 * kk + 5]);
      pa[j][kk][3] = pack_bf16x2(s[j][8 * kk + 6], s[j][8 * kk + 7]);
    }
  mbar_wait(&bar_v, 0);
  wgmma_reg_fence(o);
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < NKV; ++j) {
    const uint32_t sv = smem_u32(smem_v + j * TXT_TILE_BYTES);
#pragma unroll
    for (int kk = 0; kk < TXT_BN / 16; ++kk) {
      // V tile [128 kv x 64 hd], 128-byte rows: MN-major, 8-row k groups 1024 B apart, 16 kv rows (2048 B) per MMA
      const uint64_t dv = make_smem_desc(sv + kk * 2048, TXT_BN * 128, 1024);
      wgmma_rs_n64_tb(o, pa[j][kk], dv);
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_reg_fence(o);

  // ---- epilogue: O / l -> bf16 -> out[b * seq + q, h * 64 + ...]
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (qpos[r] >= a.seq) continue;
    __nv_bfloat16* dst = a.out + (static_cast<size_t>(b) * a.seq + qpos[r]) * a.ldo + h * TXT_HD;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i + 2 * t4) =
          pack_bf16x2(o[4 * i + 2 * r] * inv_l[r], o[4 * i + 2 * r + 1] * inv_l[r]);
  }
}

int warmup_text() {
  int rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_text_kernel<1>), TXT_SMEM_BYTES, "attn_text_kernel<1>");
  if (!rc) rc = ensure_dyn_smem(reinterpret_cast<const void*>(attn_text_kernel<2>), TXT_SMEM_BYTES, "attn_text_kernel<2>");
  return rc;
}

// ---- T5LayerNorm: one warp per row, two passes over the row (sum of squares, then scale; the second read hits L1 / L2)
__global__ void __launch_bounds__(256)
rms_norm_rows_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, const float* __restrict__ w, int rows_per_batch,
                     int row_begin, int row_count, int total, int dim, float eps) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= total) return;
  const int b = warp / row_count;
  const size_t row = static_cast<size_t>(b) * rows_per_batch + row_begin + (warp - b * row_count);
  const float4* x4 = reinterpret_cast<const float4*>(x + row * dim);
  const int nvec = dim >> 2;
  float ss = 0.f;
  for (int c = lane; c < nvec; c += 32) {
    const float4 v = x4[c];
    ss += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float r = rsqrtf(ss / static_cast<float>(dim) + eps);
  uint2* y2 = reinterpret_cast<uint2*>(y + row * dim);
  const float4* w4 = reinterpret_cast<const float4*>(w);
  for (int c = lane; c < nvec; c += 32) {
    const float4 v = x4[c];
    const float4 g = __ldg(w4 + c);
    y2[c] = make_uint2(pack_bf16x2(v.x * r * g.x, v.y * r * g.y), pack_bf16x2(v.z * r * g.z, v.w * r * g.w));
  }
}

// ---- embedding lookup: one thread per 4 columns of a row; an id outside [0, vocab) reads nothing and gives a zero row
__global__ void embed_tokens_kernel(const int* __restrict__ ids, long long rows, int rows_per_batch,
                                    const __nv_bfloat16* __restrict__ table, int vocab, int dim,
                                    const __nv_bfloat16* __restrict__ pos_table, float* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int nvec = dim >> 2;
  if (idx >= rows * nvec) return;
  const long long row = idx / nvec;
  const int c = static_cast<int>(idx - row * nvec) * 4;
  const int id = __ldg(ids + row);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (id >= 0 && id < vocab) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(table + static_cast<size_t>(id) * dim + c));
    const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
    const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
    v = make_float4(lo.x, lo.y, hi.x, hi.y);
    if (pos_table != nullptr) {
      const int p = static_cast<int>(row % rows_per_batch);
      const uint2 q = __ldg(reinterpret_cast<const uint2*>(pos_table + static_cast<size_t>(p) * dim + c));
      const float2 plo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&q.x));
      const float2 phi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&q.y));
      v.x += plo.x;
      v.y += plo.y;
      v.z += phi.x;
      v.w += phi.y;
    }
  }
  *reinterpret_cast<float4*>(out + row * dim + c) = v;
}

}  // namespace pf

extern "C" {

int pf_attn_fwd_text(const pf_attn_text_desc* d, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(d != nullptr && d->qkv != nullptr && d->out != nullptr, "pf_attn_fwd_text: null pointer");
  PF_REQUIRE(d->head_dim == TXT_HD, "pf_attn_fwd_text: head_dim %d unsupported (64 only)", d->head_dim);
  PF_REQUIRE(d->batch > 0 && d->heads > 0 && d->seq > 0, "pf_attn_fwd_text: bad shape (batch %d heads %d seq %d)", d->batch,
             d->heads, d->seq);
  PF_REQUIRE(d->seq <= TXT_MAX_SEQ, "pf_attn_fwd_text: seq %d exceeds %d", d->seq, TXT_MAX_SEQ);
  PF_REQUIRE(d->ld_qkv >= 3LL * d->heads * TXT_HD && d->ld_qkv % 8 == 0 && (reinterpret_cast<uintptr_t>(d->qkv) & 15) == 0,
             "pf_attn_fwd_text: ld_qkv %lld must be >= 3*heads*64 and a multiple of 8, qkv 16-byte aligned", (long long)d->ld_qkv);
  PF_REQUIRE(d->ldo >= static_cast<long long>(d->heads) * TXT_HD && d->ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(d->out) & 15) == 0,
             "pf_attn_fwd_text: ldo %lld must be >= heads*64 and a multiple of 8, out 16-byte aligned", (long long)d->ldo);
  CUtensorMap tm;
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(3) * d->heads * TXT_HD, static_cast<uint64_t>(d->seq),
                              static_cast<uint64_t>(d->batch)};
    const uint64_t strides[2] = {static_cast<uint64_t>(d->ld_qkv) * 2, static_cast<uint64_t>(d->ld_qkv) * 2 * d->seq};
    const uint32_t box[3] = {TXT_HD, TXT_BN, 1};
    if (int rc = encode_tensor_map(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, d->qkv, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return rc;
  }
  TextAttnArgs a{};
  a.out = static_cast<__nv_bfloat16*>(d->out);
  a.ldo = d->ldo;
  a.heads = d->heads;
  a.seq = d->seq;
  a.scale = d->scale;
  a.bias = d->bias;
  a.key_mask = d->key_mask;
  a.causal = d->causal;
  if (int rc = warmup_text()) return rc;
  const dim3 grid((d->seq + TXT_BM - 1) / TXT_BM, d->heads, d->batch);
  if (d->seq <= TXT_BN) attn_text_kernel<1><<<grid, TXT_THREADS, TXT_SMEM_BYTES, stream>>>(tm, a);
  else attn_text_kernel<2><<<grid, TXT_THREADS, TXT_SMEM_BYTES, stream>>>(tm, a);
  return check_launch("pf_attn_fwd_text");
}

int pf_rms_norm_rows(const float* x, void* y, const float* w, int32_t batches, int32_t rows_per_batch, int32_t row_begin,
                     int32_t row_count, int32_t dim, float eps, void* stream) {
  using namespace pf;
  PF_REQUIRE(x && y && w, "pf_rms_norm_rows: null pointer");
  PF_REQUIRE(dim > 0 && dim % 4 == 0, "pf_rms_norm_rows: dim=%d must be a positive multiple of 4", dim);
  // float4 loads of x and w; 8-byte stores of four bf16
  PF_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "pf_rms_norm_rows: x must be 16-byte aligned");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(w) & 15) == 0, "pf_rms_norm_rows: w must be 16-byte aligned");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(y) & 7) == 0, "pf_rms_norm_rows: y must be 8-byte aligned");
  PF_REQUIRE(batches > 0 && row_count > 0 && row_begin >= 0 && row_begin + row_count <= rows_per_batch,
             "pf_rms_norm_rows: bad row range (batches %d rows %d begin %d count %d)", batches, rows_per_batch, row_begin, row_count);
  const long long warps = static_cast<long long>(batches) * row_count;
  PF_REQUIRE(warps < (1LL << 31) - 255, "pf_rms_norm_rows: too many rows");
  rms_norm_rows_kernel<<<static_cast<int>((warps + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, static_cast<__nv_bfloat16*>(y), w, rows_per_batch, row_begin, row_count, static_cast<int>(warps), dim, eps);
  return check_launch("pf_rms_norm_rows");
}

int pf_embed_tokens(const int32_t* ids, int64_t rows, int32_t rows_per_batch, const void* table, int32_t vocab, int32_t dim,
                    const void* pos_table, int32_t max_pos, float* out, void* stream) {
  using namespace pf;
  PF_REQUIRE(ids && table && out, "pf_embed_tokens: null pointer");
  PF_REQUIRE(rows > 0 && rows_per_batch > 0 && rows % rows_per_batch == 0, "pf_embed_tokens: rows %lld must be a multiple of "
             "rows_per_batch %d", (long long)rows, rows_per_batch);
  PF_REQUIRE(vocab > 0 && dim > 0 && dim % 4 == 0, "pf_embed_tokens: vocab %d, dim %d (a positive multiple of 4)", vocab, dim);
  PF_REQUIRE(pos_table == nullptr || rows_per_batch <= max_pos, "pf_embed_tokens: rows_per_batch %d exceeds the %d positions",
             rows_per_batch, max_pos);
  PF_REQUIRE((reinterpret_cast<uintptr_t>(table) & 7) == 0 && (reinterpret_cast<uintptr_t>(pos_table) & 7) == 0 &&
                 (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "pf_embed_tokens: tables must be 8-byte and out 16-byte aligned");
  const long long total = rows * (dim / 4);
  embed_tokens_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      ids, rows, rows_per_batch, static_cast<const __nv_bfloat16*>(table), vocab, dim,
      static_cast<const __nv_bfloat16*>(pos_table), out);
  return check_launch("pf_embed_tokens");
}

}  // extern "C"
