// pf_lpips.cu — the work around the VGG16 convs of LPIPS (video_vae/modeling_lpips.py:32-45) for the VAE training step.
//
// The 13 convs of vgg16().features[:30] run on pf_causal_conv3d (kt = 1, relu / select epilogues).  Here:
//   pf_maxpool2x2 / _bwd   MaxPool2d(2, 2) on channels-last bf16, and its gradient routed to the window's first maximum in
//                          row-major order (torch's rule: `val > max || isnan(val)` scanning the window row by row);
//   pf_lpips_head_fwd      normalize_tensor (:107-110), (f0 - f1)^2, lin_k = Dropout + 1x1 Conv2d(C, 1) (:58-65), the
//                          spatial mean and the sum over the taps, per image, without an activation-sized temporary;
//   pf_lpips_tap_bwd       at one tap and one branch: the closed-form head gradient + the max-pool routing of the next
//                          slice's data gradient, under the ReLU select, rounded once to bf16;
//   pf_lpips_dropout_mask  the keep mask the head draws, for tests.
// A "lane group" of L = min(32, C/8) lanes owns one pixel; each lane holds C / (8 L) (1 or 2) 8-channel chunks, so the
// per-pixel channel sums are shuffle reductions inside the group.  Every sum has a fixed order; there are no atomics.
// Dropout is Philox4x32-10 with key = the 64-bit seed (read on the device) and counter (channel / 4, image * H * W + pixel,
// tap, 0): element kept iff (u >> 8) * 2^-24 >= p, then scaled by 1 / (1 - p).
#include <curand_philox4x32_x.h>

#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

using bf16 = __nv_bfloat16;
constexpr int LP_THREADS = 256;
constexpr int LP_WARPS = LP_THREADS / 32;
constexpr int LP_MAX_CHUNKS = 2;   // 8-channel chunks per lane: C <= 512
constexpr float LP_EPS = 1e-10f;   // normalize_tensor's eps

__device__ __forceinline__ void unpack8(const uint4 v, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

// torch's max_pool2d scan of one window: the first element greater than every earlier one (or NaN) in row-major order
__device__ __forceinline__ int window_argmax(float a0, float a1, float a2, float a3) {
  float m = -INFINITY;
  int idx = 0;
  if (a0 > m || isnan(a0)) { m = a0; idx = 0; }
  if (a1 > m || isnan(a1)) { m = a1; idx = 1; }
  if (a2 > m || isnan(a2)) { m = a2; idx = 2; }
  if (a3 > m || isnan(a3)) { m = a3; idx = 3; }
  return idx;
}

// 8 keep multipliers (0 or 1/(1-p)) of channels [c0, c0 + 8) of one pixel
__device__ __forceinline__ void dropout8(uint2 key, int c0, uint32_t pix, int tap, float p, float keep_scale, float* m) {
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const uint4 u = curand_Philox4x32_10(make_uint4(static_cast<uint32_t>(c0 / 4 + q), pix, static_cast<uint32_t>(tap), 0u), key);
    const uint32_t r[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) m[4 * q + i] = __uint2float_rz(r[i] >> 8) * 0x1p-24f >= p ? keep_scale : 0.f;
  }
}

__device__ __forceinline__ uint2 seed_key(const int64_t* seed, float p) {
  if (p <= 0.f) return make_uint2(0u, 0u);
  const uint64_t s = static_cast<uint64_t>(*seed);
  return make_uint2(static_cast<uint32_t>(s), static_cast<uint32_t>(s >> 32));
}

__device__ __forceinline__ float group_sum(float v, int L) {
  for (int o = L >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------------------ max-pool
__global__ void __launch_bounds__(LP_THREADS) maxpool2x2_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy,
                                                                bf16* __restrict__ out, int n, int h, int w, int c) {
  const int cv = c / 8, ho = h / 2, wo = w / 2;
  const long long total = static_cast<long long>(n) * ho * wo * cv;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ch = static_cast<int>(i % cv);
    long long r = i / cv;
    const int ow = static_cast<int>(r % wo);
    r /= wo;
    const int oh = static_cast<int>(r % ho);
    const long long img = r / ho;
    const size_t base = ((static_cast<size_t>(img) * h + 2 * oh) * w + 2 * ow) * c + ch * 8;
    const size_t off[4] = {0, static_cast<size_t>(c), static_cast<size_t>(w) * c, static_cast<size_t>(w) * c + c};
    uint4 v[4];
    float f[4][8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      v[k] = __ldg(reinterpret_cast<const uint4*>(x + base + off[k]));
      unpack8(v[k], f[k]);
    }
    const size_t obase = ((static_cast<size_t>(img) * ho + oh) * wo + ow) * c + ch * 8;
    uint32_t arg[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) arg[e] = window_argmax(f[0][e], f[1][e], f[2][e], f[3][e]);
    if (dy == nullptr) {
      // the winner's bf16 bits themselves (no float round trip)
      uint4 o;
      uint32_t* ow32 = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        uint32_t word = 0;
#pragma unroll
        for (int hl = 0; hl < 2; ++hl) {
          const int e = 2 * q + hl;
          const uint32_t w0 = reinterpret_cast<const uint32_t*>(&v[0])[q], w1 = reinterpret_cast<const uint32_t*>(&v[1])[q];
          const uint32_t w2 = reinterpret_cast<const uint32_t*>(&v[2])[q], w3 = reinterpret_cast<const uint32_t*>(&v[3])[q];
          const uint32_t win = arg[e] == 0 ? w0 : arg[e] == 1 ? w1 : arg[e] == 2 ? w2 : w3;
          word |= ((win >> (16 * hl)) & 0xffffu) << (16 * hl);
        }
        ow32[q] = word;
      }
      *reinterpret_cast<uint4*>(out + obase) = o;
    } else {
      const uint4 g = __ldg(reinterpret_cast<const uint4*>(dy + obase));
      const uint32_t* g32 = reinterpret_cast<const uint32_t*>(&g);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        uint4 o;
        uint32_t* o32 = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t lo = arg[2 * q] == static_cast<uint32_t>(k) ? (g32[q] & 0xffffu) : 0u;
          const uint32_t hi = arg[2 * q + 1] == static_cast<uint32_t>(k) ? (g32[q] & 0xffff0000u) : 0u;
          o32[q] = lo | hi;
        }
        *reinterpret_cast<uint4*>(out + base + off[k]) = o;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------- head
struct LpTap {
  const bf16* f0;
  const bf16* f1;
  const float* lin;
  int c, h, w;
};

struct LpHeadArgs {
  LpTap tap[PF_LPIPS_MAX_TAPS];
  int n, taps;
  float p, keep_scale;
  const int64_t* seed;
  float* partial;   // [taps, n, PF_LPIPS_HEAD_BLOCKS]
  float* val;       // [n]
};

__host__ __device__ __forceinline__ int lane_group(int c) { return c / 8 < 32 ? c / 8 : 32; }

// grid (PF_LPIPS_HEAD_BLOCKS, n, taps): block b sums the pixels [HW b / NB, HW (b+1) / NB) of one (image, tap)
__global__ void __launch_bounds__(LP_THREADS) lpips_head_fwd_kernel(const LpHeadArgs a) {
  const int blk = blockIdx.x, img = blockIdx.y, k = blockIdx.z;
  const LpTap t = a.tap[k];
  const int hw = t.h * t.w;
  const int L = lane_group(t.c), nch = t.c / (8 * L);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane % L, gpw = 32 / L;
  const int p0 = static_cast<int>(static_cast<long long>(hw) * blk / PF_LPIPS_HEAD_BLOCKS);
  const int p1 = static_cast<int>(static_cast<long long>(hw) * (blk + 1) / PF_LPIPS_HEAD_BLOCKS);
  const uint2 key = seed_key(a.seed, a.p);
  float wl[LP_MAX_CHUNKS][8];
#pragma unroll
  for (int j = 0; j < LP_MAX_CHUNKS; ++j)
#pragma unroll
    for (int e = 0; e < 8; ++e) wl[j][e] = j < nch ? __ldg(t.lin + 8 * (sub + j * L) + e) : 0.f;
  float acc = 0.f;
  // the trip count is uniform over the warp (the shuffles need every lane); a group past p1 contributes zeros
  for (int pb = p0 + warp * gpw; pb < p1; pb += LP_WARPS * gpw) {
    const int p = pb + lane / L;
    const bool valid = p < p1;
    const size_t pix = static_cast<size_t>(img) * hw + (valid ? p : p0);
    float f0[LP_MAX_CHUNKS][8], f1[LP_MAX_CHUNKS][8];
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < LP_MAX_CHUNKS; ++j) {
      if (j < nch && valid) {
        unpack8(__ldg(reinterpret_cast<const uint4*>(t.f0 + pix * t.c + 8 * (sub + j * L))), f0[j]);
        unpack8(__ldg(reinterpret_cast<const uint4*>(t.f1 + pix * t.c + 8 * (sub + j * L))), f1[j]);
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) f0[j][e] = f1[j][e] = 0.f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        s0 = fmaf(f0[j][e], f0[j][e], s0);
        s1 = fmaf(f1[j][e], f1[j][e], s1);
      }
    }
    s0 = group_sum(s0, L);
    s1 = group_sum(s1, L);
    const float i0 = 1.f / (sqrtf(s0) + LP_EPS), i1 = 1.f / (sqrtf(s1) + LP_EPS);
#pragma unroll
    for (int j = 0; j < LP_MAX_CHUNKS; ++j) {
      if (j >= nch || !valid) continue;
      float m[8];
      if (a.p > 0.f) dropout8(key, 8 * (sub + j * L), static_cast<uint32_t>(pix), k, a.p, a.keep_scale, m);
      else
#pragma unroll
        for (int e = 0; e < 8; ++e) m[e] = 1.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = f0[j][e] * i0 - f1[j][e] * i1;
        acc = fmaf(wl[j][e] * m[e], d * d, acc);
      }
    }
  }
  // fixed-order block sum: xor tree in the warp, then the warps in order
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float ws[LP_WARPS];
  if (lane == 0) ws[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < LP_WARPS; ++i) s += ws[i];
    a.partial[(static_cast<size_t>(k) * a.n + img) * PF_LPIPS_HEAD_BLOCKS + blk] = s;
  }
}

__global__ void lpips_head_reduce_kernel(const LpHeadArgs a) {
  const int img = blockIdx.x * blockDim.x + threadIdx.x;
  if (img >= a.n) return;
  float v = 0.f;
  for (int k = 0; k < a.taps; ++k) {
    const float* part = a.partial + (static_cast<size_t>(k) * a.n + img) * PF_LPIPS_HEAD_BLOCKS;
    float s = 0.f;
    for (int b = 0; b < PF_LPIPS_HEAD_BLOCKS; ++b) s += part[b];
    v += s / static_cast<float>(a.tap[k].h * a.tap[k].w);
  }
  a.val[img] = v;
}

// ------------------------------------------------------------------------------------------------------- tap backward
struct LpBwdArgs {
  const bf16* f;        // this branch's tap (ReLU output), [n, h, w, c]
  const bf16* fo;       // the other branch's tap
  const float* lin;
  const bf16* dnext;    // [n, h/2, w/2, c] or null
  const float* grad;    // [n]
  const int64_t* seed;
  bf16* dz;
  int n, h, w, c, tap;
  float p, keep_scale;
};

// With u = f / (|f| + eps), the head's value at a pixel is (1/HW) sum_c w_c m_c (u_c - uo_c)^2, so with
// a_c = 2 g / HW * w_c m_c (u_c - uo_c):  df_j = a_j / (|f| + eps) - f_j (sum_c a_c f_c) / (|f| (|f| + eps)^2), and 0 where
// |f| = 0 (torch's sqrt backward is 0/0 there; the ReLU select drops it in the reference).
__global__ void __launch_bounds__(LP_THREADS) lpips_tap_bwd_kernel(const LpBwdArgs a) {
  const int hw = a.h * a.w;
  const int L = lane_group(a.c), nch = a.c / (8 * L);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane % L, gpw = 32 / L;
  const long long items = static_cast<long long>(a.n) * hw;
  const uint2 key = seed_key(a.seed, a.p);
  const int wo = a.w / 2;
  const size_t rowc = static_cast<size_t>(a.w) * a.c;
  float wl[LP_MAX_CHUNKS][8];
#pragma unroll
  for (int j = 0; j < LP_MAX_CHUNKS; ++j)
#pragma unroll
    for (int e = 0; e < 8; ++e) wl[j][e] = j < nch ? __ldg(a.lin + 8 * (sub + j * L) + e) : 0.f;
  for (long long ib = (static_cast<long long>(blockIdx.x) * LP_WARPS + warp) * gpw; ib < items;
       ib += static_cast<long long>(gridDim.x) * LP_WARPS * gpw) {
    const long long i = ib + lane / L;
    const bool valid = i < items;
    const long long ii = valid ? i : ib;
    const int img = static_cast<int>(ii / hw), r = static_cast<int>(ii % hw);
    // with a next slice, the groups of a warp walk the 2x2 windows (the four pixels of a window are neighbours in i)
    int hh, ww, s = 0;
    if (a.dnext != nullptr) {
      const int win = r >> 2;
      s = r & 3;
      hh = 2 * (win / wo) + (s >> 1);
      ww = 2 * (win % wo) + (s & 1);
    } else {
      hh = r / a.w;
      ww = r - hh * a.w;
    }
    const size_t pix = static_cast<size_t>(img) * hw + static_cast<size_t>(hh) * a.w + ww;
    const float gs = 2.f * __ldg(a.grad + img) / static_cast<float>(hw);
    float f[LP_MAX_CHUNKS][8], fo[LP_MAX_CHUNKS][8];
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < LP_MAX_CHUNKS; ++j) {
      if (j < nch) {
        unpack8(__ldg(reinterpret_cast<const uint4*>(a.f + pix * a.c + 8 * (sub + j * L))), f[j]);
        unpack8(__ldg(reinterpret_cast<const uint4*>(a.fo + pix * a.c + 8 * (sub + j * L))), fo[j]);
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[j][e] = fo[j][e] = 0.f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        s0 = fmaf(f[j][e], f[j][e], s0);
        s1 = fmaf(fo[j][e], fo[j][e], s1);
      }
    }
    s0 = group_sum(s0, L);
    s1 = group_sum(s1, L);
    const float n0 = sqrtf(s0);
    const float i0 = 1.f / (n0 + LP_EPS), i1 = 1.f / (sqrtf(s1) + LP_EPS);
    float av[LP_MAX_CHUNKS][8];
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < LP_MAX_CHUNKS; ++j) {
      float m[8];
      if (a.p > 0.f && j < nch) dropout8(key, 8 * (sub + j * L), static_cast<uint32_t>(pix), a.tap, a.p, a.keep_scale, m);
      else
#pragma unroll
        for (int e = 0; e < 8; ++e) m[e] = 1.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        av[j][e] = gs * wl[j][e] * m[e] * (f[j][e] * i0 - fo[j][e] * i1);
        dot = fmaf(av[j][e], f[j][e], dot);
      }
    }
    dot = group_sum(dot, L);
    const float coef = n0 > 0.f ? dot / (n0 * (n0 + LP_EPS) * (n0 + LP_EPS)) : 0.f;
    const float ai = n0 > 0.f ? i0 : 0.f;
    if (!valid) continue;
#pragma unroll
    for (int j = 0; j < LP_MAX_CHUNKS; ++j) {
      if (j >= nch) continue;
      const int c0 = 8 * (sub + j * L);
      float route[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) route[e] = 0.f;
      if (a.dnext != nullptr) {
        const size_t wbase = (static_cast<size_t>(img) * a.h + (hh & ~1)) * rowc + static_cast<size_t>(ww & ~1) * a.c + c0;
        float q[4][8], dn[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(a.f + wbase)), q[0]);
        unpack8(__ldg(reinterpret_cast<const uint4*>(a.f + wbase + a.c)), q[1]);
        unpack8(__ldg(reinterpret_cast<const uint4*>(a.f + wbase + rowc)), q[2]);
        unpack8(__ldg(reinterpret_cast<const uint4*>(a.f + wbase + rowc + a.c)), q[3]);
        const size_t nb = ((static_cast<size_t>(img) * (a.h / 2) + (hh >> 1)) * wo + (ww >> 1)) * a.c + c0;
        unpack8(__ldg(reinterpret_cast<const uint4*>(a.dnext + nb)), dn);
#pragma unroll
        for (int e = 0; e < 8; ++e) route[e] = window_argmax(q[0][e], q[1][e], q[2][e], q[3][e]) == s ? dn[e] : 0.f;
      }
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float head = av[j][e] * ai - f[j][e] * coef;
        o[e] = f[j][e] > 0.f ? head + route[e] : 0.f;
      }
      uint4 u;
      u.x = pack_bf16x2(o[0], o[1]); u.y = pack_bf16x2(o[2], o[3]); u.z = pack_bf16x2(o[4], o[5]); u.w = pack_bf16x2(o[6], o[7]);
      *reinterpret_cast<uint4*>(a.dz + pix * a.c + c0) = u;
    }
  }
}

__global__ void lpips_dropout_mask_kernel(const int64_t* seed, int tap, long long pixels, int c, float p, uint8_t* mask) {
  const uint2 key = seed_key(seed, p);
  const int cv = c / 8;
  const long long total = pixels * cv;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = i / cv;
    const int c0 = static_cast<int>(i % cv) * 8;
    float m[8];
    dropout8(key, c0, static_cast<uint32_t>(pix), tap, p, 1.f, m);
    uint2 out;
    out.x = (m[0] != 0.f) | ((m[1] != 0.f) << 8) | ((m[2] != 0.f) << 16) | ((m[3] != 0.f) << 24);
    out.y = (m[4] != 0.f) | ((m[5] != 0.f) << 8) | ((m[6] != 0.f) << 16) | ((m[7] != 0.f) << 24);
    *reinterpret_cast<uint2*>(mask + pix * c + c0) = out;
  }
}

static int elementwise_grid(long long work) {
  int sms = num_sms();
  if (sms <= 0) sms = 132;
  const long long blocks = (work + LP_THREADS - 1) / LP_THREADS;
  return static_cast<int>(blocks < 16LL * sms ? (blocks > 0 ? blocks : 1) : 16LL * sms);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int lp_check_channels(int c, const char* what) {
  PF_REQUIRE(c == 64 || c == 128 || c == 256 || c == 512, "%s: channels=%d must be 64, 128, 256 or 512 (VGG16)", what, c);
  return 0;
}

static int lp_check_pixels(long long n, long long h, long long w, const char* what) {
  PF_REQUIRE(n > 0 && h > 0 && w > 0, "%s: bad shape", what);
  PF_REQUIRE(n * h * w < (1LL << 31), "%s: %lld pixels are too many", what, n * h * w);
  return 0;
}

static int maxpool_run(const void* x, const void* dy, void* out, int n, int h, int w, int c, void* stream, const char* what) {
  PF_REQUIRE(x && out, "%s: null pointer", what);
  if (int rc = lp_check_pixels(n, h, w, what)) return rc;
  PF_REQUIRE(h % 2 == 0 && w % 2 == 0, "%s: h=%d and w=%d must be even", what, h, w);
  PF_REQUIRE(c > 0 && c % 8 == 0, "%s: channels=%d must be a multiple of 8", what, c);
  PF_REQUIRE(aligned16(x) && aligned16(out) && (!dy || aligned16(dy)), "%s: tensors must be 16-byte aligned", what);
  const long long work = static_cast<long long>(n) * (h / 2) * (w / 2) * (c / 8);
  maxpool2x2_kernel<<<elementwise_grid(work), LP_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const bf16*>(x), static_cast<const bf16*>(dy), static_cast<bf16*>(out), n, h, w, c);
  return check_launch(what);
}

static int dropout_check(float p, const int64_t* seed, const char* what) {
  PF_REQUIRE(p >= 0.f && p < 1.f, "%s: dropout p=%g must be in [0, 1)", what, static_cast<double>(p));
  PF_REQUIRE(p == 0.f || seed != nullptr, "%s: dropout needs the seed tensor", what);
  return 0;
}

}  // namespace pf

extern "C" int pf_maxpool2x2(const void* x, void* y, int32_t n, int32_t h, int32_t w, int32_t c, void* stream) {
  return pf::maxpool_run(x, nullptr, y, n, h, w, c, stream, "pf_maxpool2x2");
}

extern "C" int pf_maxpool2x2_bwd(const void* x, const void* dy, void* dx, int32_t n, int32_t h, int32_t w, int32_t c,
                                 void* stream) {
  PF_REQUIRE(dy != nullptr, "pf_maxpool2x2_bwd: null pointer");
  return pf::maxpool_run(x, dy, dx, n, h, w, c, stream, "pf_maxpool2x2_bwd");
}

extern "C" int pf_lpips_head_fwd(const pf_lpips_head_desc* d, void* stream) {
  using namespace pf;
  PF_REQUIRE(d != nullptr && d->val != nullptr && d->workspace != nullptr, "pf_lpips_head_fwd: null pointer");
  PF_REQUIRE(d->n > 0 && d->n < 65536, "pf_lpips_head_fwd: n=%d images must be in [1, 65535]", d->n);
  PF_REQUIRE(d->taps >= 1 && d->taps <= PF_LPIPS_MAX_TAPS, "pf_lpips_head_fwd: taps=%d must be in [1, %d]", d->taps,
             PF_LPIPS_MAX_TAPS);
  if (int rc = dropout_check(d->p, d->seed, "pf_lpips_head_fwd")) return rc;
  PF_REQUIRE(d->workspace_floats >= static_cast<int64_t>(d->taps) * d->n * PF_LPIPS_HEAD_BLOCKS,
             "pf_lpips_head_fwd: workspace of %lld floats is too small (taps * n * %d)",
             static_cast<long long>(d->workspace_floats), PF_LPIPS_HEAD_BLOCKS);
  LpHeadArgs a{};
  for (int k = 0; k < d->taps; ++k) {
    PF_REQUIRE(d->f0[k] && d->f1[k] && d->lin[k], "pf_lpips_head_fwd: null pointer at tap %d", k);
    PF_REQUIRE(aligned16(d->f0[k]) && aligned16(d->f1[k]), "pf_lpips_head_fwd: tap %d features must be 16-byte aligned", k);
    if (int rc = lp_check_channels(d->c[k], "pf_lpips_head_fwd")) return rc;
    if (int rc = lp_check_pixels(d->n, d->h[k], d->w[k], "pf_lpips_head_fwd")) return rc;
    a.tap[k] = LpTap{static_cast<const bf16*>(d->f0[k]), static_cast<const bf16*>(d->f1[k]), d->lin[k], d->c[k], d->h[k], d->w[k]};
  }
  a.n = d->n;
  a.taps = d->taps;
  a.p = d->p;
  a.keep_scale = 1.f / (1.f - d->p);
  a.seed = d->seed;
  a.partial = d->workspace;
  a.val = d->val;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  lpips_head_fwd_kernel<<<dim3(PF_LPIPS_HEAD_BLOCKS, d->n, d->taps), LP_THREADS, 0, st>>>(a);
  if (int rc = check_launch("pf_lpips_head_fwd")) return rc;
  lpips_head_reduce_kernel<<<(d->n + 127) / 128, 128, 0, st>>>(a);
  return check_launch("pf_lpips_head_fwd (reduce)");
}

extern "C" int pf_lpips_tap_bwd(const pf_lpips_tap_bwd_desc* d, void* stream) {
  using namespace pf;
  PF_REQUIRE(d != nullptr && d->f && d->f_other && d->lin && d->grad && d->dz, "pf_lpips_tap_bwd: null pointer");
  if (int rc = lp_check_channels(d->c, "pf_lpips_tap_bwd")) return rc;
  if (int rc = lp_check_pixels(d->n, d->h, d->w, "pf_lpips_tap_bwd")) return rc;
  PF_REQUIRE(d->tap >= 0 && d->tap < PF_LPIPS_MAX_TAPS, "pf_lpips_tap_bwd: tap=%d must be in [0, %d)", d->tap,
             PF_LPIPS_MAX_TAPS);
  if (int rc = dropout_check(d->p, d->seed, "pf_lpips_tap_bwd")) return rc;
  PF_REQUIRE(!d->d_next || (d->h % 2 == 0 && d->w % 2 == 0), "pf_lpips_tap_bwd: the max-pool route needs even h and w");
  PF_REQUIRE(aligned16(d->f) && aligned16(d->f_other) && aligned16(d->dz) && (!d->d_next || aligned16(d->d_next)),
             "pf_lpips_tap_bwd: tensors must be 16-byte aligned");
  LpBwdArgs a{};
  a.f = static_cast<const bf16*>(d->f);
  a.fo = static_cast<const bf16*>(d->f_other);
  a.lin = d->lin;
  a.dnext = static_cast<const bf16*>(d->d_next);
  a.grad = d->grad;
  a.seed = d->seed;
  a.dz = static_cast<bf16*>(d->dz);
  a.n = d->n; a.h = d->h; a.w = d->w; a.c = d->c; a.tap = d->tap;
  a.p = d->p;
  a.keep_scale = 1.f / (1.f - d->p);
  const int gpw = 32 / lane_group(d->c);
  const long long warps = (static_cast<long long>(d->n) * d->h * d->w + gpw - 1) / gpw;
  lpips_tap_bwd_kernel<<<elementwise_grid(warps * 32), LP_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(a);
  return check_launch("pf_lpips_tap_bwd");
}

extern "C" int pf_lpips_dropout_mask(const int64_t* seed, int32_t tap, int32_t n, int32_t h, int32_t w, int32_t c, float p,
                                     uint8_t* mask, void* stream) {
  using namespace pf;
  PF_REQUIRE(seed && mask, "pf_lpips_dropout_mask: null pointer");
  if (int rc = lp_check_channels(c, "pf_lpips_dropout_mask")) return rc;
  if (int rc = lp_check_pixels(n, h, w, "pf_lpips_dropout_mask")) return rc;
  PF_REQUIRE(tap >= 0 && tap < PF_LPIPS_MAX_TAPS, "pf_lpips_dropout_mask: tap=%d must be in [0, %d)", tap, PF_LPIPS_MAX_TAPS);
  if (int rc = dropout_check(p, seed, "pf_lpips_dropout_mask")) return rc;
  PF_REQUIRE((reinterpret_cast<uintptr_t>(mask) & 7) == 0, "pf_lpips_dropout_mask: mask must be 8-byte aligned");
  const long long pixels = static_cast<long long>(n) * h * w;
  lpips_dropout_mask_kernel<<<elementwise_grid(pixels * (c / 8)), LP_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      seed, tap, pixels, c, p, mask);
  return check_launch("pf_lpips_dropout_mask");
}
