// pf_elementwise.cu — the HBM-bound kernels of the DiT step: LayerNorm+AdaLN modulate pre-pass, the small-M linear
// (all-layer AdaLN modulation GEMV + conditioning MLPs), timestep sinusoid, patchify / unpatchify, CFG+Euler.
// Reference op sites are cited in include/pf_b200.h next to each entry point.
#include <cuda_fp8.h>

#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

// ---------------------------------------------------------------------------------------------------------------
// LN + modulate: one warp per row, row kept in registers (dim <= 2048, dim % 128 == 0), 128-bit loads, 64-bit stores.
// Algorithmic traffic: 4 B (fp32 in) + 2 B (bf16 out) per element; with the e4m3 output (FP8) 4 B + 1 B, and the row's amax
// is one more warp reduction over the values already in registers (pf_b200.h FP8 contract).
// ---------------------------------------------------------------------------------------------------------------
constexpr int LN_MAX_VEC = 16;  // float4 per lane
constexpr float E4M3_MAX = 448.f;

// e4m3 bytes of (a, b, c, d) * inv, packed little-endian (pf_b200.h FP8 contract)
__device__ __forceinline__ uint32_t e4m3x4(float a, float b, float c, float d, float inv) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a * inv, b * inv), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c * inv, d * inv), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <bool FP8>
__global__ void __launch_bounds__(256)
ln_modulate_kernel(const float* __restrict__ x, void* __restrict__ y_, float* __restrict__ row_scale, int batches,
                   int rows_per_batch, int row_begin, int row_count, int dim, const float* __restrict__ shift,
                   const float* __restrict__ scale, long long mod_batch_stride, float eps) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int total = batches * row_count;
  if (warp >= total) return;
  const int b = warp / row_count;
  const int r = warp - b * row_count;
  const size_t row = static_cast<size_t>(b) * rows_per_batch + row_begin + r;
  const int nvec = dim >> 7;  // float4 per lane
  const float4* x4 = reinterpret_cast<const float4*>(x + row * dim);

  float4 v[LN_MAX_VEC];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    if (i < nvec) {
      v[i] = x4[i * 32 + lane];
      sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / static_cast<float>(dim);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    if (i < nvec) {
      const float a = v[i].x - mean, bq = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      ss += (a * a + bq * bq) + (c * c + d * d);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rstd = rsqrtf(ss / static_cast<float>(dim) + eps);

  const float4* sh4 = reinterpret_cast<const float4*>(shift + b * mod_batch_stride);
  const float4* sc4 = reinterpret_cast<const float4*>(scale + b * mod_batch_stride);
  if constexpr (!FP8) {
    uint2* y2 = reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(y_) + row * dim);
#pragma unroll
    for (int i = 0; i < LN_MAX_VEC; ++i) {
      if (i < nvec) {
        const float4 sh = __ldg(sh4 + i * 32 + lane);
        const float4 sc = __ldg(sc4 + i * 32 + lane);
        const float o0 = (v[i].x - mean) * rstd * (1.f + sc.x) + sh.x;
        const float o1 = (v[i].y - mean) * rstd * (1.f + sc.y) + sh.y;
        const float o2 = (v[i].z - mean) * rstd * (1.f + sc.z) + sh.z;
        const float o3 = (v[i].w - mean) * rstd * (1.f + sc.w) + sh.w;
        y2[i * 32 + lane] = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
      }
    }
  } else {
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < LN_MAX_VEC; ++i) {
      if (i < nvec) {
        const float4 sh = __ldg(sh4 + i * 32 + lane);
        const float4 sc = __ldg(sc4 + i * 32 + lane);
        v[i].x = (v[i].x - mean) * rstd * (1.f + sc.x) + sh.x;
        v[i].y = (v[i].y - mean) * rstd * (1.f + sc.y) + sh.y;
        v[i].z = (v[i].z - mean) * rstd * (1.f + sc.z) + sh.z;
        v[i].w = (v[i].w - mean) * rstd * (1.f + sc.w) + sh.w;
        amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[i].x), fabsf(v[i].y)), fmaxf(fabsf(v[i].z), fabsf(v[i].w))));
      }
    }
    amax = warp_max(amax);
    const float inv = amax > 0.f ? E4M3_MAX / amax : 0.f;
    uint32_t* y4 = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(y_) + row * dim);
#pragma unroll
    for (int i = 0; i < LN_MAX_VEC; ++i)
      if (i < nvec) y4[i * 32 + lane] = e4m3x4(v[i].x, v[i].y, v[i].z, v[i].w, inv);
    if (lane == 0) row_scale[row] = amax / E4M3_MAX;
  }
}

// Row quantiser bf16 -> e4m3 + row scale (pf_b200.h FP8 contract): one warp per row, two passes over the row (amax, then
// quantise; the second read is served by L1 / L2), 16-byte loads and 8-byte stores.  cols % 8 == 0.
__global__ void __launch_bounds__(256)
quantize_rows_fp8_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, uint8_t* __restrict__ y, long long ldy,
                         float* __restrict__ row_scale, int rows_per_batch, int row_begin, int row_count, int total, int cols) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= total) return;
  const int b = warp / row_count;
  const size_t row = static_cast<size_t>(b) * rows_per_batch + row_begin + (warp - b * row_count);
  const uint4* x8 = reinterpret_cast<const uint4*>(x + row * ldx);
  uint2* y8 = reinterpret_cast<uint2*>(y + row * ldy);
  const int nchunk = cols >> 3;
  auto unpack = [](const uint4& u, float (&f)[8]) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 p = __bfloat1622float2(h[i]);
      f[2 * i] = p.x;
      f[2 * i + 1] = p.y;
    }
  };
  float amax = 0.f;
  for (int c = lane; c < nchunk; c += 32) {
    float f[8];
    unpack(x8[c], f);
#pragma unroll
    for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(f[i]));
  }
  amax = warp_max(amax);
  const float inv = amax > 0.f ? E4M3_MAX / amax : 0.f;
  for (int c = lane; c < nchunk; c += 32) {
    float f[8];
    unpack(x8[c], f);
    y8[c] = make_uint2(e4m3x4(f[0], f[1], f[2], f[3], inv), e4m3x4(f[4], f[5], f[6], f[7], inv));
  }
  if (lane == 0) row_scale[row] = amax / E4M3_MAX;
}

// ---------------------------------------------------------------------------------------------------------------
// small-M linear: one warp per output column n, all m rows at once; W row streamed once with 128-bit loads.
// Algorithmic traffic: 2*K bytes per output column (weights dominate; x is staged in shared memory).
// ---------------------------------------------------------------------------------------------------------------
constexpr int SL_MAX_M = 8;

template <int M>
__global__ void __launch_bounds__(256)
small_linear_kernel(const float* __restrict__ x, int k, const __nv_bfloat16* __restrict__ w,
                    const float* __restrict__ bias, int n, float* __restrict__ y, int act_in, int act_out,
                    int accumulate, int round_in_bf16) {
  extern __shared__ float xs[];  // [M, k]
  for (int i = threadIdx.x; i < M * k; i += blockDim.x) {
    float v = x[i];
    if (act_in == 1) v = silu_f(v);
    if (round_in_bf16) v = __bfloat162float(__float2bfloat16(v));
    xs[i] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int col = blockIdx.x * (blockDim.x >> 5) + warp;
  if (col >= n) return;
  const uint4* w4 = reinterpret_cast<const uint4*>(w + static_cast<size_t>(col) * k);
  float acc[M];
#pragma unroll
  for (int m = 0; m < M; ++m) acc[m] = 0.f;
  const int nchunk = k >> 3;
  for (int c = lane; c < nchunk; c += 32) {
    const uint4 u = __ldg(w4 + c);
    float wf[8];
    {
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __bfloat1622float2(h[i]);
        wf[2 * i] = f.x;
        wf[2 * i + 1] = f.y;
      }
    }
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const float4 a = *reinterpret_cast<const float4*>(xs + m * k + c * 8);
      const float4 bq = *reinterpret_cast<const float4*>(xs + m * k + c * 8 + 4);
      acc[m] += wf[0] * a.x + wf[1] * a.y + wf[2] * a.z + wf[3] * a.w + wf[4] * bq.x + wf[5] * bq.y + wf[6] * bq.z +
                wf[7] * bq.w;
    }
  }
#pragma unroll
  for (int m = 0; m < M; ++m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], o);
  }
  if (lane == 0) {
    const float bv = bias ? bias[col] : 0.f;
#pragma unroll
    for (int m = 0; m < M; ++m) {
      float v = acc[m] + bv;
      if (act_out == 1) v = silu_f(v);
      float* dst = y + static_cast<size_t>(m) * n + col;
      *dst = accumulate ? (*dst + v) : v;
    }
  }
}

__global__ void timestep_embedding_kernel(const float* __restrict__ t, int m, int dim, float* __restrict__ out,
                                          int round_bf16) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim >> 1;
  if (idx >= m * half) return;
  const int r = idx / half;
  const int i = idx - r * half;
  // exponent = -ln(10000) * i / half   (downscale_freq_shift = 0), fp32 like the reference (E:47-53)
  const float freq = expf(-9.210340371976184f * static_cast<float>(i) / static_cast<float>(half));
  const float arg = t[r] * freq;
  float c = cosf(arg), s = sinf(arg);
  if (round_bf16) {
    c = __bfloat162float(__float2bfloat16(c));
    s = __bfloat162float(__float2bfloat16(s));
  }
  out[static_cast<size_t>(r) * dim + i] = c;         // flip_sin_to_cos: cos first
  out[static_cast<size_t>(r) * dim + half + i] = s;
}

template <typename T>
__global__ void patchify_kernel(const T* __restrict__ lat, int B, int C, int T_, int H, int W,
                                __nv_bfloat16* __restrict__ tok, int rows_per_batch, int tok_begin) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int hh = H >> 1, ww = W >> 1;
  const int feat = 4 * C;
  const long long total = static_cast<long long>(B) * T_ * hh * ww * feat;
  if (idx >= total) return;
  const int f = static_cast<int>(idx % feat);
  long long rest = idx / feat;
  const int xw = static_cast<int>(rest % ww);
  rest /= ww;
  const int yh = static_cast<int>(rest % hh);
  rest /= hh;
  const int tt = static_cast<int>(rest % T_);
  const int b = static_cast<int>(rest / T_);
  const int c = f % C;
  const int p = f / C;
  const int p1 = p >> 1, p2 = p & 1;
  const size_t src = (((static_cast<size_t>(b) * C + c) * T_ + tt) * H + (2 * yh + p1)) * W + (2 * xw + p2);
  const size_t row = static_cast<size_t>(b) * rows_per_batch + tok_begin + (static_cast<size_t>(tt) * hh + yh) * ww + xw;
  tok[row * feat + f] = __float2bfloat16(static_cast<float>(lat[src]));
}

template <typename T>
__global__ void unpatchify_kernel(const float* __restrict__ x, int rows_per_batch, int row_begin, int B, int C, int T_,
                                  int H, int W, T* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * C * T_ * H * W;
  if (idx >= total) return;
  const int xw = static_cast<int>(idx % W);
  long long rest = idx / W;
  const int yh = static_cast<int>(rest % H);
  rest /= H;
  const int tt = static_cast<int>(rest % T_);
  rest /= T_;
  const int c = static_cast<int>(rest % C);
  const int b = static_cast<int>(rest / C);
  const int hh = H >> 1, ww = W >> 1;
  const int feat = 4 * C;
  const size_t row = static_cast<size_t>(b) * rows_per_batch + row_begin + (static_cast<size_t>(tt) * hh + (yh >> 1)) * ww + (xw >> 1);
  const int f = (((yh & 1) << 1) | (xw & 1)) * C + c;
  out[idx] = static_cast<T>(x[row * feat + f]);
}

__global__ void cfg_euler_kernel(const float* __restrict__ v2, float guidance, float dsigma,
                                 const float* __restrict__ x, float* __restrict__ x_out, long long n) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float vu = v2[i], vc = v2[n + i];
  const float v = vu + guidance * (vc - vu);
  x_out[i] = x[i] + dsigma * v;
}

// Stage hop of the pyramidal sampler (P:729-743): out[.., 2i+di, 2j+dj] = alpha * x[.., i, j] + beta * n[.., 2i+di, 2j+dj], where
// every 2x2 block of n ~ N(0, (1+gamma) I - gamma 1 1^T) (sample_block_noise, P:697-703) is L z with z the block's four iid
// normals (z_in, same layout as out) and L the Cholesky factor of the 4x4 covariance.  One thread per 2x2 block.
template <typename T>
__global__ void stage_hop_kernel(const T* __restrict__ x, const float* __restrict__ z, T* __restrict__ out, long long planes,
                                 int h, int w, float alpha, float beta, float4 l0, float4 l1, float4 l2, float4 l3) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = planes * h * w;
  if (idx >= total) return;
  const int j = static_cast<int>(idx % w);
  const int i = static_cast<int>((idx / w) % h);
  const long long p = idx / (static_cast<long long>(w) * h);
  const float xv = alpha * static_cast<float>(x[idx]);
  const long long o = (p * 2 * h + 2 * i) * (2 * w) + 2 * j;
  const float2 za = *reinterpret_cast<const float2*>(z + o);              // block order (di, dj): (0,0), (0,1), (1,0), (1,1)
  const float2 zb = *reinterpret_cast<const float2*>(z + o + 2 * w);
  const float n0 = l0.x * za.x;
  const float n1 = l1.x * za.x + l1.y * za.y;
  const float n2 = l2.x * za.x + l2.y * za.y + l2.z * zb.x;
  const float n3 = l3.x * za.x + l3.y * za.y + l3.z * zb.x + l3.w * zb.y;
  out[o] = static_cast<T>(xv + beta * n0);
  out[o + 1] = static_cast<T>(xv + beta * n1);
  out[o + 2 * w] = static_cast<T>(xv + beta * n2);
  out[o + 2 * w + 1] = static_cast<T>(xv + beta * n3);
}

}  // namespace pf

extern "C" {

int pf_stage_hop(const void* x, int32_t x_is_f32, const float* z, void* out, int64_t planes, int32_t h, int32_t w, float alpha,
                 float beta, const float* chol16, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(x && z && out && chol16 && planes > 0 && h > 0 && w > 0, "pf_stage_hop: bad arguments");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(z) & 7) == 0, "pf_stage_hop: z must be 8-byte aligned");
  const float4 l0 = make_float4(chol16[0], chol16[1], chol16[2], chol16[3]);
  const float4 l1 = make_float4(chol16[4], chol16[5], chol16[6], chol16[7]);
  const float4 l2 = make_float4(chol16[8], chol16[9], chol16[10], chol16[11]);
  const float4 l3 = make_float4(chol16[12], chol16[13], chol16[14], chol16[15]);
  const long long total = planes * h * w;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  if (x_is_f32)
    stage_hop_kernel<float><<<blocks, 256, 0, stream>>>(static_cast<const float*>(x), z, static_cast<float*>(out), planes, h, w,
                                                         alpha, beta, l0, l1, l2, l3);
  else
    stage_hop_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), z,
                                                                 static_cast<__nv_bfloat16*>(out), planes, h, w, alpha, beta,
                                                                 l0, l1, l2, l3);
  return check_launch("pf_stage_hop");
}

int pf_ln_modulate(const float* x, void* y, int32_t batches, int32_t rows_per_batch, int32_t row_begin,
                   int32_t row_count, int32_t dim, const float* shift, const float* scale, int64_t mod_batch_stride,
                   float eps, void* stream) {
  using namespace pf;
  PF_REQUIRE(x && y && shift && scale, "pf_ln_modulate: null pointer");
  PF_REQUIRE(dim % 128 == 0 && dim <= 128 * LN_MAX_VEC, "pf_ln_modulate: dim=%d must be a multiple of 128 and <= %d", dim, 128 * LN_MAX_VEC);
  PF_REQUIRE(batches > 0 && row_count > 0 && row_begin >= 0 && row_begin + row_count <= rows_per_batch, "pf_ln_modulate: bad row range");
  PF_REQUIRE(mod_batch_stride % 4 == 0, "pf_ln_modulate: modulation stride must be a multiple of 4 floats");
  // float4 loads of x, shift and scale; 8-byte stores of four bf16
  PF_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "pf_ln_modulate: x must be 16-byte aligned");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(shift) & 15) == 0, "pf_ln_modulate: shift must be 16-byte aligned");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(scale) & 15) == 0, "pf_ln_modulate: scale must be 16-byte aligned");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(y) & 7) == 0, "pf_ln_modulate: y must be 8-byte aligned");
  const long long warps = static_cast<long long>(batches) * row_count;
  const int blocks = static_cast<int>((warps + 7) / 8);
  ln_modulate_kernel<false><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, y, nullptr, batches, rows_per_batch, row_begin, row_count, dim, shift, scale, mod_batch_stride, eps);
  return check_launch("pf_ln_modulate");
}

int pf_ln_modulate_fp8(const float* x, void* y, float* row_scale, int32_t batches, int32_t rows_per_batch, int32_t row_begin,
                       int32_t row_count, int32_t dim, const float* shift, const float* scale, int64_t mod_batch_stride,
                       float eps, void* stream) {
  using namespace pf;
  PF_REQUIRE(x && y && row_scale && shift && scale, "pf_ln_modulate_fp8: null pointer");
  PF_REQUIRE(dim % 128 == 0 && dim <= 128 * LN_MAX_VEC, "pf_ln_modulate_fp8: dim=%d must be a multiple of 128 and <= %d", dim, 128 * LN_MAX_VEC);
  PF_REQUIRE(batches > 0 && row_count > 0 && row_begin >= 0 && row_begin + row_count <= rows_per_batch, "pf_ln_modulate_fp8: bad row range");
  PF_REQUIRE(mod_batch_stride % 4 == 0, "pf_ln_modulate_fp8: modulation stride must be a multiple of 4 floats");
  // float4 loads of x, shift and scale; 4-byte stores of four e4m3
  PF_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "pf_ln_modulate_fp8: x must be 16-byte aligned");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(shift) & 15) == 0, "pf_ln_modulate_fp8: shift must be 16-byte aligned");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(scale) & 15) == 0, "pf_ln_modulate_fp8: scale must be 16-byte aligned");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(y) & 3) == 0, "pf_ln_modulate_fp8: y must be 4-byte aligned");
  PF_REQUIRE((reinterpret_cast<uintptr_t>(row_scale) & 3) == 0, "pf_ln_modulate_fp8: row_scale must be 4-byte aligned");
  const long long warps = static_cast<long long>(batches) * row_count;
  const int blocks = static_cast<int>((warps + 7) / 8);
  ln_modulate_kernel<true><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, y, row_scale, batches, rows_per_batch, row_begin, row_count, dim, shift, scale, mod_batch_stride, eps);
  return check_launch("pf_ln_modulate_fp8");
}

int pf_quantize_rows_fp8(const void* x, int64_t ldx, void* y, int64_t ldy, float* row_scale, int32_t batches,
                         int32_t rows_per_batch, int32_t row_begin, int32_t row_count, int32_t cols, void* stream) {
  using namespace pf;
  PF_REQUIRE(x && y && row_scale, "pf_quantize_rows_fp8: null pointer");
  PF_REQUIRE(cols > 0 && cols % 8 == 0, "pf_quantize_rows_fp8: cols=%d must be a positive multiple of 8", cols);
  PF_REQUIRE(ldx % 8 == 0 && ldx >= cols && ldy % 8 == 0 && ldy >= cols,
             "pf_quantize_rows_fp8: ldx=%lld and ldy=%lld must be >= cols and multiples of 8", (long long)ldx, (long long)ldy);
  PF_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 7) == 0,
             "pf_quantize_rows_fp8: x must be 16-byte and y 8-byte aligned");
  PF_REQUIRE(batches > 0 && row_count > 0 && row_begin >= 0 && row_begin + row_count <= rows_per_batch,
             "pf_quantize_rows_fp8: bad row range (batches %d rows %d begin %d count %d)", batches, rows_per_batch, row_begin,
             row_count);
  const long long warps = static_cast<long long>(batches) * row_count;
  PF_REQUIRE(warps < (1LL << 31) - 255, "pf_quantize_rows_fp8: too many rows");
  const int blocks = static_cast<int>((warps + 7) / 8);
  quantize_rows_fp8_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), ldx, static_cast<uint8_t*>(y), ldy, row_scale, rows_per_batch, row_begin,
      row_count, static_cast<int>(warps), cols);
  return check_launch("pf_quantize_rows_fp8");
}

int pf_small_linear(const float* x, int32_t m, int32_t k, const void* w, const float* bias, int32_t n, float* y,
                    int32_t act_in, int32_t act_out, int32_t accumulate, int32_t round_in_bf16, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(x && w && y, "pf_small_linear: null pointer");
  PF_REQUIRE(m >= 1 && m <= SL_MAX_M, "pf_small_linear: m=%d must be in [1, %d]", m, SL_MAX_M);
  PF_REQUIRE(k % 8 == 0 && k > 0, "pf_small_linear: k=%d must be a multiple of 8", k);
  PF_REQUIRE(n > 0, "pf_small_linear: n=%d must be positive", n);
  PF_REQUIRE(4LL * m * k <= 96 * 1024, "pf_small_linear: m*k too large for shared memory");
  const int smem = m * k * 4;
  PF_REQUIRE((reinterpret_cast<uintptr_t>(w) & 15) == 0, "pf_small_linear: w must be 16-byte aligned (16-byte loads)");
  const int blocks = (n + 7) / 8;
#define PF_SL_CASE(MM)                                                                                          \
  case MM: {                                                                                                    \
    auto kern = small_linear_kernel<MM>;                                                                        \
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);   \
    kern<<<blocks, 256, smem, stream>>>(x, k, static_cast<const __nv_bfloat16*>(w), bias, n, y, act_in, act_out, \
                                        accumulate, round_in_bf16);                                             \
    break;                                                                                                      \
  }
  switch (m) {
    PF_SL_CASE(1)
    PF_SL_CASE(2)
    PF_SL_CASE(3)
    PF_SL_CASE(4)
    PF_SL_CASE(5)
    PF_SL_CASE(6)
    PF_SL_CASE(7)
    PF_SL_CASE(8)
  }
#undef PF_SL_CASE
  return check_launch("pf_small_linear");
}

int pf_timestep_embedding(const float* t, int32_t m, int32_t dim, float* out, int32_t round_bf16, void* stream) {
  using namespace pf;
  PF_REQUIRE(t && out && m > 0 && dim > 0 && dim % 2 == 0, "pf_timestep_embedding: bad arguments");
  const int total = m * (dim / 2);
  timestep_embedding_kernel<<<(total + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(t, m, dim, out,
                                                                                                  round_bf16);
  return check_launch("pf_timestep_embedding");
}

int pf_patchify(const void* latent, int32_t latent_is_f32, int32_t b, int32_t c, int32_t t, int32_t h, int32_t w,
                void* tokens, int32_t rows_per_batch, int32_t tok_begin, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(latent && tokens && h % 2 == 0 && w % 2 == 0, "pf_patchify: bad arguments");
  PF_REQUIRE(b > 0 && c > 0 && t > 0 && h > 0 && w > 0, "pf_patchify: b=%d c=%d t=%d h=%d w=%d must be positive", b, c, t, h, w);
  PF_REQUIRE(tok_begin >= 0 && tok_begin + static_cast<long long>(t) * (h / 2) * (w / 2) <= rows_per_batch,
             "pf_patchify: token range exceeds rows_per_batch");
  const long long total = static_cast<long long>(b) * c * t * h * w;
  const int blocks = static_cast<int>((total + 255) / 256);
  if (latent_is_f32)
    patchify_kernel<float><<<blocks, 256, 0, stream>>>(static_cast<const float*>(latent), b, c, t, h, w,
                                                       static_cast<__nv_bfloat16*>(tokens), rows_per_batch, tok_begin);
  else
    patchify_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(latent), b, c, t, h,
                                                               w, static_cast<__nv_bfloat16*>(tokens), rows_per_batch,
                                                               tok_begin);
  return check_launch("pf_patchify");
}

int pf_unpatchify(const float* x, int32_t rows_per_batch, int32_t row_begin, int32_t b, int32_t c, int32_t t,
                  int32_t h, int32_t w, void* out, int32_t out_is_f32, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(x && out && h % 2 == 0 && w % 2 == 0, "pf_unpatchify: bad arguments");
  PF_REQUIRE(b > 0 && c > 0 && t > 0 && h > 0 && w > 0, "pf_unpatchify: b=%d c=%d t=%d h=%d w=%d must be positive", b, c, t, h, w);
  PF_REQUIRE(row_begin >= 0, "pf_unpatchify: row_begin=%d must be >= 0", row_begin);
  PF_REQUIRE(row_begin + static_cast<long long>(t) * (h / 2) * (w / 2) <= rows_per_batch,
             "pf_unpatchify: token range [row_begin %d, +t*(h/2)*(w/2)) exceeds rows_per_batch %d", row_begin, rows_per_batch);
  const long long total = static_cast<long long>(b) * c * t * h * w;
  const int blocks = static_cast<int>((total + 255) / 256);
  if (out_is_f32)
    unpatchify_kernel<float><<<blocks, 256, 0, stream>>>(x, rows_per_batch, row_begin, b, c, t, h, w,
                                                         static_cast<float*>(out));
  else
    unpatchify_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(x, rows_per_batch, row_begin, b, c, t, h, w,
                                                                 static_cast<__nv_bfloat16*>(out));
  return check_launch("pf_unpatchify");
}

int pf_cfg_euler_step(const float* v2, float guidance, float dsigma, const float* x, float* x_out, int64_t n,
                      void* stream) {
  using namespace pf;
  PF_REQUIRE(v2 && x && x_out && n > 0, "pf_cfg_euler_step: bad arguments");
  cfg_euler_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      v2, guidance, dsigma, x, x_out, n);
  return check_launch("pf_cfg_euler_step");
}

}  // extern "C"
