// pf_groupnorm.cuh — per-frame GroupNorm device code shared by the inference kernels (pf_vae_elementwise.cu) and the
// training kernels (pf_groupnorm_train.cu): one definition of the statistics' partial sums, of their finalisation and of
// the affine + SiLU, so a bf16 channels-last frame gets the same bits from both.
#pragma once

#include "pf_common.cuh"

namespace pf {

// Frames are split into this many voxel ranges for the partial sums.  It depends on the frame size only, never on how
// many frames a call holds: per-frame statistics are bitwise identical whatever the temporal chunking.
__host__ __device__ inline int gn_splits(long long voxels) {
  long long nsplit = (voxels + 4095) / 4096;
  if (nsplit < 1) nsplit = 1;
  if (nsplit > 64) nsplit = 64;
  return static_cast<int>(nsplit);
}

__device__ __forceinline__ float gn_load1(const __nv_bfloat16* p) { return __bfloat162float(*p); }
__device__ __forceinline__ float gn_load1(const float* p) { return __ldg(p); }

// 8 consecutive elements (16-byte aligned)
__device__ __forceinline__ void gn_load8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void gn_load8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ void gn_store1(__nv_bfloat16* p, float v) { *p = __float2bfloat16(v); }
__device__ __forceinline__ void gn_store1(float* p, float v) { *p = v; }
__device__ __forceinline__ void gn_store8(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 w;
  w.x = pack_bf16x2(v[0], v[1]);
  w.y = pack_bf16x2(v[2], v[3]);
  w.z = pack_bf16x2(v[4], v[5]);
  w.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = w;
}
__device__ __forceinline__ void gn_store8(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}

// The normalised, affine output and its optional SiLU: act((x - mean) * rstd * gamma + beta).
__device__ __forceinline__ float gn_affine_act(float x, float mean, float rstd, float gamma, float beta, int silu) {
  float v = (x - mean) * rstd * gamma + beta;
  if (silu) v = silu_f(v);
  return v;
}

// Statistics, pass 1, for one (frame, voxel range) of a channels-last frame `base` [voxels][channels]: per channel, the
// fp32 sum and sum of squares of x - K over voxels [v0, v1), with the pivot K = x[voxel 0, channel].  Unshifted fp32 sums
// lose the variance to cancellation in E[x^2] - mean^2 once a group's |mean| is large against its std (~4% rstd error at
// |mean|/std = 100); shifted by a value inside the channel's own distribution they stay accurate.  Every thread reads the
// same pivot, so the sums are deterministic and independent of how frames are split across calls.  Each thread owns one
// 8-channel vector position and strides over voxels; the per-thread partials are parked in shared memory
// `sh` [vstep][channels][2] and summed in a fixed order into out [channels][2].
template <typename T>
__device__ __forceinline__ void gn_partial_frame(const T* __restrict__ base, int channels, long long v0, long long v1,
                                                 float* __restrict__ out, float* sh) {
  const int cvecs = channels >> 3;
  const int cv = threadIdx.x % cvecs;
  const int vlane = threadIdx.x / cvecs;
  const int vstep = blockDim.x / cvecs;
  float s[8], ss[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = ss[i] = 0.f;
  if (vlane < vstep) {
    float k[8];
    gn_load8(base + cv * 8, k);
    for (long long v = v0 + vlane; v < v1; v += vstep) {
      float f[8];
      gn_load8(base + v * channels + cv * 8, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = f[i] - k[i];   // exact for bf16 operands within 2^16 of each other
        s[i] += d;
        ss[i] += d * d;
      }
    }
    float* dst = sh + (static_cast<size_t>(vlane) * channels + cv * 8) * 2;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      dst[2 * i] = s[i];
      dst[2 * i + 1] = ss[i];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * channels; i += blockDim.x) {
    float acc = 0.f;
    for (int l = 0; l < vstep; ++l) acc += sh[static_cast<size_t>(l) * channels * 2 + i];
    out[i] = acc;
  }
}

// Statistics, pass 2: (mean, rstd) of group g of one frame, combined in double.  partial: the frame's [nsplit][channels][2]
// shifted sums; pivot + c * pivot_cstride: channel c's pivot.  Per channel, S = sum(x - K) and SS = sum((x - K)^2) give
// sum(x) = S + nK and sum(x^2) = SS + 2KS + nK^2.
template <typename T>
__device__ __forceinline__ void gn_finalize_group(const T* pivot, long long pivot_cstride, const float* __restrict__ partial,
                                                  int nsplit, int channels, int g, int cpg, long long voxels, float eps,
                                                  float* __restrict__ out) {
  const double nv = static_cast<double>(voxels);
  double s = 0.0, ss = 0.0;
  for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
    double sc = 0.0, ssc = 0.0;
    for (int sp = 0; sp < nsplit; ++sp) {
      const float* p = partial + (static_cast<size_t>(sp) * channels + c) * 2;
      sc += p[0];
      ssc += p[1];
    }
    const double k = gn_load1(pivot + c * pivot_cstride);
    s += sc + nv * k;
    ss += ssc + 2.0 * k * sc + nv * k * k;
  }
  const double n = nv * cpg;
  const double mean = s / n;
  double var = ss / n - mean * mean;
  if (var < 0.0) var = 0.0;
  out[0] = static_cast<float>(mean);
  out[1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
}

}  // namespace pf
