// pf_attn_pack.cu — one stage's head-major q / k / v for the masked attention, with the reference's RoPE, and its backward.
//
// Memory-bound: every source element is read once and every packed element written once.  A thread owns 8 consecutive
// columns of one (batch, packed row, head); threads are ordered (row, head, column chunk) so that a warp reads whole source
// rows (the heads of a row are adjacent in the Linear / qk-norm outputs) and the row's 512-byte RoPE table is shared through
// L1 by all its heads.  The entries and their argument checks are in pf_api.cu (include/pf_b200.h pf_attn_stage_pack).
#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

namespace {

constexpr int PACK_HD = 64;
constexpr int PACK_THREADS = 256;

__device__ __forceinline__ void load8(const void* src, bool f32, float (&x)[8]) {
  if (f32) {
    const float4 a = reinterpret_cast<const float4*>(src)[0];
    const float4 b = reinterpret_cast<const float4*>(src)[1];
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w;
    x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
  } else {
    const uint4 u = *reinterpret_cast<const uint4*>(src);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(h[i]);
      x[2 * i] = f.x;
      x[2 * i + 1] = f.y;
    }
  }
}

__device__ __forceinline__ void store8(void* dst, bool f32, const float (&x)[8]) {
  if (f32) {
    reinterpret_cast<float4*>(dst)[0] = make_float4(x[0], x[1], x[2], x[3]);
    reinterpret_cast<float4*>(dst)[1] = make_float4(x[4], x[5], x[6], x[7]);
  } else {
    uint4 u;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
    *reinterpret_cast<uint4*>(dst) = u;
  }
}

// kBwd = false: sources -> packed (RoPE on q, k).  kBwd = true: packed gradients -> source gradients (transposed RoPE).
template <bool kBwd>
__global__ void __launch_bounds__(PACK_THREADS) attn_stage_pack_kernel(const pf_attn_pack_desc d) {
  const int seq = d.text_len + d.rows;
  const int i = blockIdx.x * PACK_THREADS + threadIdx.x;
  if (i >= seq * d.heads * 8) return;
  const int b = blockIdx.y;
  const int chunk = i & 7;
  const int h = (i >> 3) % d.heads;
  const int s = (i >> 3) / d.heads;
  const bool is_text = s < d.text_len;

  float f[16];
  if (d.freqs != nullptr) {
    // pairs 4 chunk .. 4 chunk + 3 of the row's [32, 2, 2] table: f[4 p + 2 c + j] multiplies x[2 p + j] into out[2 p + c]
    const float4* fr = reinterpret_cast<const float4*>(d.freqs + b * d.freqs_batch_stride + s * d.freqs_row_stride + chunk * 16);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 v = fr[j];
      f[4 * j] = v.x; f[4 * j + 1] = v.y; f[4 * j + 2] = v.z; f[4 * j + 3] = v.w;
    }
  }
  const int64_t packed_off = ((static_cast<int64_t>(b) * d.heads + h) * seq + s) * PACK_HD + chunk * 8;

#pragma unroll
  for (int t = 0; t < 3; ++t) {
    char* src;
    bool f32;
    if (is_text) {
      const int64_t* st = d.text_strides[t];
      f32 = d.text_f32[t] != 0;
      src = static_cast<char*>(d.text[t]) +
            ((static_cast<int64_t>(b) * d.n_stages + d.stage) * st[0] + s * st[1] + h * st[2] + chunk * 8) * (f32 ? 4 : 2);
    } else {
      const int64_t* st = d.video_strides[t];
      f32 = d.video_f32[t] != 0;
      src = static_cast<char*>(d.video[t]) +
            (b * st[0] + static_cast<int64_t>(d.row0 + s - d.text_len) * st[1] + h * st[2] + chunk * 8) * (f32 ? 4 : 2);
    }
    __nv_bfloat16* packed = static_cast<__nv_bfloat16*>(d.packed[t]) + packed_off;
    float x[8], y[8];
    load8(kBwd ? static_cast<const void*>(packed) : src, kBwd ? false : f32, x);
    if (t < 2 && d.freqs != nullptr) {
#pragma unroll
      for (int p = 0; p < 4; ++p) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          if (kBwd)   // d x[2p + c] = g[2p] f[p][0][c] + g[2p + 1] f[p][1][c] (autograd's mul + sum_to_size)
            y[2 * p + c] = __fadd_rn(__fmul_rn(x[2 * p], f[4 * p + c]), __fmul_rn(x[2 * p + 1], f[4 * p + 2 + c]));
          else        // out[2p + c] = f[p][c][0] x[2p] + f[p][c][1] x[2p + 1] (apply_rope, no contraction)
            y[2 * p + c] = __fadd_rn(__fmul_rn(f[4 * p + 2 * c], x[2 * p]), __fmul_rn(f[4 * p + 2 * c + 1], x[2 * p + 1]));
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = x[j];
    }
    store8(kBwd ? static_cast<void*>(src) : static_cast<void*>(packed), kBwd ? f32 : false, y);
  }
}

}  // namespace

// Launch only: the descriptor is validated by the C entries (pf_api.cu).
int attn_stage_pack_launch(const pf_attn_pack_desc* d, bool bwd, cudaStream_t stream) {
  const int64_t threads = static_cast<int64_t>(d->text_len + d->rows) * d->heads * 8;
  const dim3 grid(static_cast<unsigned>((threads + PACK_THREADS - 1) / PACK_THREADS), static_cast<unsigned>(d->batch));
  if (bwd) {
    attn_stage_pack_kernel<true><<<grid, PACK_THREADS, 0, stream>>>(*d);
    return check_launch("pf_attn_stage_pack_bwd");
  }
  attn_stage_pack_kernel<false><<<grid, PACK_THREADS, 0, stream>>>(*d);
  return check_launch("pf_attn_stage_pack");
}

}  // namespace pf
