// pf_groupnorm_train.cu — trainable per-frame GroupNorm (+ SiLU) of the causal video VAE: forward and backward on bf16 or
// fp32 activations, read in place in two layout forms.
//
// Replaces the autograd of CausalGroupNorm.forward (reference video_vae/modeling_causal_conv.py:36-43: GroupNorm over
// (channels of a group) x H x W of every (batch, frame)) and of the SiLU that follows it in CausalResnetBlock3D
// (video_vae/modeling_resnet.py:127-143) and in the encoder's / decoder's conv_norm_out -> conv_act
// (video_vae/modeling_enc_dec.py:194-195, 362-363).
//
//   forms  : channel form -- x[b, c, t, h, w] at b*sb + t*st + (h*W + w)*C + c (channels_last_3d): one thread owns 8
//            consecutive channels of a voxel, 16-byte loads along C;  plane form -- at b*sb + c*sc + t*st + h*W + w (every
//            (b, c, t) plane contiguous, e.g. NCDHW): one warp owns a channel's plane, 16-byte loads along the voxels where
//            the strides allow, element loads otherwise.
//   forward: partial sums per (frame, split, channel) about a per-channel pivot (the inference statistics' device code,
//            pf_groupnorm.cuh), combined per (frame, group) in double into stats [frames, groups, 2] = (mean, rstd); then
//            y = act((x - mean) * rstd * gamma + beta), dense in x's form (a bf16 y with the inference apply's SiLU, an
//            fp32 y evaluated in double, rounded once).
//   backward: z = xhat * gamma + beta recomputed, dz = dy * SiLU'(z) (or dy); pass 1 writes per (frame, split, channel)
//            fp32 sums of dz and dz * xhat; a finalize turns them into per (frame, group) A = mean(gamma dz),
//            B = mean(gamma dz xhat) (double), and a fixed-order reduce over (frame, split) gives dbeta = sum dz and
//            dgamma = sum dz xhat; pass 2 writes dx = rstd * (gamma dz - A - xhat B) in x's dtype, dense in x's form.
// No atomics anywhere: every sum has an order fixed by the shape.
#include "../../include/pf_b200.h"
#include "pf_groupnorm.cuh"

namespace pf {

constexpr int GT_THREADS = 256;
constexpr int GT_FORM_CHANNEL = 1, GT_FORM_PLANE = 2;

struct GnArgs {
  const void* x;
  const void* dy;
  void* out;                  // y (forward) or dx (backward), dense in x's form
  long long xs[3], ds[3];     // element strides of x's / dy's (b, c, t); the voxel stride is C (channel) or 1 (plane)
  int b, c, t, groups, cpg, silu, nsplit;
  long long voxels;
  float eps;
  const float* stats;         // [frames, groups, 2] (mean, rstd)
  const float* coef;          // [frames, groups, 2] (A, B)
  const float* gamma;
  const float* beta;
  float* partial;             // [frames, nsplit, c, 2]
};

// 1 + e^-z >= 1: the approximate reciprocal is within an ulp and has no slow path
__device__ __forceinline__ float gt_sigmoid(float z) { return rcp_approx_f(1.f + expf(-z)); }

// the forward's output value: a bf16 output runs the inference apply's expression (gn_affine_act: the same bits as
// pf_groupnorm_apply); an fp32 output, where fp32 rounding of the affine and the SiLU would show, is evaluated in double
// and rounded once
template <typename To>
__device__ __forceinline__ float gt_out(float x, float mean, float rstd, float gamma, float beta, int silu) {
  if (sizeof(To) == 2) return gn_affine_act(x, mean, rstd, gamma, beta, silu);
  const double z = (static_cast<double>(x) - mean) * rstd * gamma + beta;
  return static_cast<float>(silu ? z / (1.0 + exp(-z)) : z);
}

// dL/dz from dL/dact: dy * SiLU'(z) = dy * s (1 + z (1 - s)), s = sigmoid(z); dy itself without the SiLU
__device__ __forceinline__ float gt_dz(float dy, float z, int silu) {
  if (!silu) return dy;
  const float s = gt_sigmoid(z);
  return dy * s * (1.f + z * (1.f - s));
}

// ---------------------------------------------------------------------------------------------------------- channel form
// forward statistics, pass 1: one block per (frame, split), the inference kernel's per-frame body
template <typename T>
__global__ void __launch_bounds__(GT_THREADS) gt_stats_cl_kernel(const GnArgs a) {
  extern __shared__ float sh[];
  const int frame = blockIdx.x / a.nsplit, split = blockIdx.x - frame * a.nsplit;
  const int bb = frame / a.t, tt = frame - bb * a.t;
  const T* base = static_cast<const T*>(a.x) + bb * a.xs[0] + tt * a.xs[2];
  gn_partial_frame(base, a.c, a.voxels * split / a.nsplit, a.voxels * (split + 1) / a.nsplit,
                   a.partial + (static_cast<size_t>(frame) * a.nsplit + split) * a.c * 2, sh);
}

// backward pass 1: per (frame, split, channel) sums of dz and dz * xhat.  Block (frame x split, slice) owns the channels
// [64 slice, +64) (fewer in a last partial slice); its threads hold 8 channels each and stride over the split's voxels,
// accumulating in double (a thread adds up to a few hundred voxels); the per-thread sums are parked in shared memory
// [vstep][64][2] and added in a fixed order.
constexpr int GT_SLICE = 64;
template <typename Tx, typename Td>
__global__ void __launch_bounds__(GT_THREADS) gt_bwd_partial_cl_kernel(const GnArgs a) {
  __shared__ double shd[GT_THREADS / (GT_SLICE / 8) * GT_SLICE * 2];
  const int frame = blockIdx.x / a.nsplit, split = blockIdx.x - frame * a.nsplit;
  const int bb = frame / a.t, tt = frame - bb * a.t;
  const int c0 = blockIdx.y * GT_SLICE, nc = min(GT_SLICE, a.c - c0);
  const int cvecs = nc >> 3;
  const int cv = threadIdx.x % cvecs, vlane = threadIdx.x / cvecs, vstep = blockDim.x / cvecs;
  const long long v0 = a.voxels * split / a.nsplit, v1 = a.voxels * (split + 1) / a.nsplit;
  double s[8], sx[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = sx[i] = 0.0;
  if (vlane < vstep) {
    const Tx* xb = static_cast<const Tx*>(a.x) + bb * a.xs[0] + tt * a.xs[2] + c0 + cv * 8;
    const Td* db = static_cast<const Td*>(a.dy) + bb * a.ds[0] + tt * a.ds[2] + c0 + cv * 8;
    float mean[8], rstd[8], gam[8], bet[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = c0 + cv * 8 + i;
      const float* st = a.stats + 2 * (static_cast<size_t>(frame) * a.groups + c / a.cpg);
      mean[i] = __ldg(st);
      rstd[i] = __ldg(st + 1);
      gam[i] = __ldg(a.gamma + c);
      bet[i] = __ldg(a.beta + c);
    }
    for (long long v = v0 + vlane; v < v1; v += vstep) {
      float xv[8], dv[8];
      gn_load8(xb + v * a.c, xv);
      gn_load8(db + v * a.c, dv);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xh = (xv[i] - mean[i]) * rstd[i];
        const float dz = gt_dz(dv[i], xh * gam[i] + bet[i], a.silu);
        s[i] += dz;
        sx[i] += static_cast<double>(dz) * xh;
      }
    }
    double* dst = shd + (vlane * nc + cv * 8) * 2;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      dst[2 * i] = s[i];
      dst[2 * i + 1] = sx[i];
    }
  }
  __syncthreads();
  float* out = a.partial + ((static_cast<size_t>(frame) * a.nsplit + split) * a.c + c0) * 2;
  for (int i = threadIdx.x; i < 2 * nc; i += blockDim.x) {
    double acc = 0.0;
    for (int l = 0; l < vstep; ++l) acc += shd[l * nc * 2 + i];
    out[i] = static_cast<float>(acc);
  }
}

// forward apply (BWD = false: out = act(z)) or backward pass 2 (BWD = true: out = dx); grid (voxel chunks, frames), one
// thread per 8 channels of a voxel; out is dense channels-last [frames, voxels, c]
template <bool BWD, typename Tx, typename Td, typename To>
__global__ void __launch_bounds__(GT_THREADS) gt_elem_cl_kernel(const GnArgs a) {
  const int cvecs = a.c >> 3;
  const long long i = static_cast<long long>(blockIdx.x) * GT_THREADS + threadIdx.x;
  if (i >= a.voxels * cvecs) return;
  const int frame = blockIdx.y;
  const int bb = frame / a.t, tt = frame - bb * a.t;
  const int cv = static_cast<int>(i % cvecs);
  const long long v = i / cvecs;
  float xv[8], dv[8];
  gn_load8(static_cast<const Tx*>(a.x) + bb * a.xs[0] + tt * a.xs[2] + v * a.c + cv * 8, xv);
  if (BWD) gn_load8(static_cast<const Td*>(a.dy) + bb * a.ds[0] + tt * a.ds[2] + v * a.c + cv * 8, dv);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = cv * 8 + k;
    const size_t sg = 2 * (static_cast<size_t>(frame) * a.groups + c / a.cpg);
    const float mean = __ldg(a.stats + sg), rstd = __ldg(a.stats + sg + 1);
    if (!BWD) {
      xv[k] = gt_out<To>(xv[k], mean, rstd, __ldg(a.gamma + c), __ldg(a.beta + c), a.silu);
    } else {
      const float g = __ldg(a.gamma + c);
      const float xh = (xv[k] - mean) * rstd;
      const float dz = gt_dz(dv[k], xh * g + __ldg(a.beta + c), a.silu);
      xv[k] = rstd * (g * dz - __ldg(a.coef + sg) - xh * __ldg(a.coef + sg + 1));
    }
  }
  gn_store8(static_cast<To*>(a.out) + (static_cast<size_t>(frame) * a.voxels + v) * a.c + cv * 8, xv);
}

// ------------------------------------------------------------------------------------------------------------ plane form
// Statistics (BWD = false) or backward pass 1 (BWD = true), one block per (frame, split), one warp per channel at a time:
// the lanes stride over the split's voxels of the channel's plane (VEC: 8 voxels per 16-byte load) with double sums, and
// the warp's sums are combined by a fixed butterfly.
template <bool BWD, bool VEC, typename Tx, typename Td>
__global__ void __launch_bounds__(GT_THREADS) gt_partial_pl_kernel(const GnArgs a) {
  const int frame = blockIdx.x / a.nsplit, split = blockIdx.x - frame * a.nsplit;
  const int bb = frame / a.t, tt = frame - bb * a.t;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n = VEC ? a.voxels / 8 : a.voxels;
  const long long i0 = n * split / a.nsplit, i1 = n * (split + 1) / a.nsplit;
  for (int c = warp; c < a.c; c += GT_THREADS / 32) {
    const Tx* xp = static_cast<const Tx*>(a.x) + bb * a.xs[0] + c * a.xs[1] + tt * a.xs[2];
    const Td* dp = static_cast<const Td*>(a.dy) + bb * a.ds[0] + c * a.ds[1] + tt * a.ds[2];
    float k = 0.f, mean = 0.f, rstd = 0.f, gam = 0.f, bet = 0.f;
    if (!BWD) {
      k = gn_load1(xp);
    } else {
      const float* st = a.stats + 2 * (static_cast<size_t>(frame) * a.groups + c / a.cpg);
      mean = __ldg(st);
      rstd = __ldg(st + 1);
      gam = __ldg(a.gamma + c);
      bet = __ldg(a.beta + c);
    }
    double s = 0.0, s2 = 0.0;
    for (long long i = i0 + lane; i < i1; i += 32) {
      constexpr int N = VEC ? 8 : 1;
      float xv[8], dv[8];
      if (VEC) {
        gn_load8(xp + i * 8, xv);
        if (BWD) gn_load8(dp + i * 8, dv);
      } else {
        xv[0] = gn_load1(xp + i);
        if (BWD) dv[0] = gn_load1(dp + i);
      }
#pragma unroll
      for (int e = 0; e < N; ++e) {
        if (!BWD) {
          const double d = static_cast<double>(xv[e]) - k;
          s += d;
          s2 += d * d;
        } else {
          const float xh = (xv[e] - mean) * rstd;
          const float dz = gt_dz(dv[e], xh * gam + bet, a.silu);
          s += dz;
          s2 += static_cast<double>(dz) * xh;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) {
      float* out = a.partial + ((static_cast<size_t>(frame) * a.nsplit + split) * a.c + c) * 2;
      out[0] = static_cast<float>(s);
      out[1] = static_cast<float>(s2);
    }
  }
}

// forward apply / backward pass 2 in plane form: grid (planes b*c*t, voxel chunks); out is dense [b, c, t, voxels]
template <bool BWD, bool VEC, typename Tx, typename Td, typename To>
__global__ void __launch_bounds__(GT_THREADS) gt_elem_pl_kernel(const GnArgs a) {
  const long long n = VEC ? a.voxels / 8 : a.voxels;
  const int plane = blockIdx.x;
  const int tt = plane % a.t, r = plane / a.t;
  const int c = r % a.c, bb = r / a.c;
  const int frame = bb * a.t + tt;
  const size_t sg = 2 * (static_cast<size_t>(frame) * a.groups + c / a.cpg);
  const float mean = __ldg(a.stats + sg), rstd = __ldg(a.stats + sg + 1);
  const float g = __ldg(a.gamma + c), be = __ldg(a.beta + c);
  const float ca = BWD ? __ldg(a.coef + sg) : 0.f, cb = BWD ? __ldg(a.coef + sg + 1) : 0.f;
  const Tx* xp = static_cast<const Tx*>(a.x) + bb * a.xs[0] + c * a.xs[1] + tt * a.xs[2];
  const Td* dp = static_cast<const Td*>(a.dy) + bb * a.ds[0] + c * a.ds[1] + tt * a.ds[2];
  To* op = static_cast<To*>(a.out) + static_cast<size_t>(plane) * a.voxels;
  auto f = [&](float xv, float dv) {
    if (!BWD) return gt_out<To>(xv, mean, rstd, g, be, a.silu);
    const float xh = (xv - mean) * rstd;
    const float dz = gt_dz(dv, xh * g + be, a.silu);
    return rstd * (g * dz - ca - xh * cb);
  };
  // grid.y is capped at 65535 chunks of GT_THREADS: larger planes are walked in strides of the whole grid
  for (long long i = static_cast<long long>(blockIdx.y) * GT_THREADS + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.y) * GT_THREADS) {
    if (VEC) {
      float xv[8], dv[8];
      gn_load8(xp + i * 8, xv);
      if (BWD) gn_load8(dp + i * 8, dv);
#pragma unroll
      for (int e = 0; e < 8; ++e) xv[e] = f(xv[e], BWD ? dv[e] : 0.f);
      gn_store8(op + i * 8, xv);
    } else {
      gn_store1(op + i, f(gn_load1(xp + i), BWD ? gn_load1(dp + i) : 0.f));
    }
  }
}

// ------------------------------------------------------------------------------------------------------------- finalize
template <typename T>
__global__ void gt_finalize_kernel(const GnArgs a, float* __restrict__ stats) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.b * a.t * a.groups) return;
  const int frame = idx / a.groups, g = idx - frame * a.groups;
  const int bb = frame / a.t, tt = frame - bb * a.t;
  gn_finalize_group(static_cast<const T*>(a.x) + bb * a.xs[0] + tt * a.xs[2], a.xs[1],
                    a.partial + static_cast<size_t>(frame) * a.nsplit * a.c * 2, a.nsplit, a.c, g, a.cpg, a.voxels, a.eps,
                    stats + 2 * idx);
}

// backward: A = mean(gamma dz), B = mean(gamma dz xhat) per (frame, group), from the per-split channel sums, in double
__global__ void gt_bwd_coef_kernel(const GnArgs a, float* __restrict__ coef) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.b * a.t * a.groups) return;
  const int frame = idx / a.groups, g = idx - frame * a.groups;
  double sa = 0.0, sb = 0.0;
  for (int c = g * a.cpg; c < (g + 1) * a.cpg; ++c) {
    double s = 0.0, sx = 0.0;
    for (int sp = 0; sp < a.nsplit; ++sp) {
      const float* p = a.partial + ((static_cast<size_t>(frame) * a.nsplit + sp) * a.c + c) * 2;
      s += p[0];
      sx += p[1];
    }
    const double gam = a.gamma[c];
    sa += gam * s;
    sb += gam * sx;
  }
  const double n = static_cast<double>(a.voxels) * a.cpg;
  coef[2 * idx] = static_cast<float>(sa / n);
  coef[2 * idx + 1] = static_cast<float>(sb / n);
}

// dbeta[c] = sum of dz, dgamma[c] = sum of dz xhat over (frame, split) in order, in double
__global__ void gt_param_grad_kernel(const GnArgs a, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.c) return;
  const long long rows = static_cast<long long>(a.b) * a.t * a.nsplit;
  double s = 0.0, sx = 0.0;
  for (long long r = 0; r < rows; ++r) {
    const float* p = a.partial + (r * a.c + c) * 2;
    s += p[0];
    sx += p[1];
  }
  if (dbeta) dbeta[c] = static_cast<float>(s);
  if (dgamma) dgamma[c] = static_cast<float>(sx);
}

// --------------------------------------------------------------------------------------------------------------- host
// The layout form of a [b, c, t, h, w] tensor with element strides s_in; strides of size-1 axes are never used and are
// taken as 0.  Channel form also needs every 8-channel vector 16-byte aligned.
static int gt_form(const void* p, const int64_t* s_in, int b, int c, int t, int h, int w, long long (&s)[5]) {
  const int n[5] = {b, c, t, h, w};
  for (int i = 0; i < 5; ++i) s[i] = n[i] == 1 ? 0 : s_in[i];
  const bool chan = s[1] == 1 && (w == 1 || s[4] == c) && (h == 1 || s[3] == static_cast<long long>(w) * c) &&
                    s[0] % 8 == 0 && s[2] % 8 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0;
  if (chan) return GT_FORM_CHANNEL;
  const bool plane = (w == 1 || s[4] == 1) && (h == 1 || s[3] == w);
  return plane ? GT_FORM_PLANE : 0;
}

struct GtPlan {
  GnArgs a;
  int form, x_f32, t2_f32, vec;   // t2: the output's dtype (forward) or dy's (backward)
  long long ws_need;
};

static int gt_plan(const pf_groupnorm_train_desc* d, bool bwd, GtPlan& p) {
  PF_REQUIRE(d != nullptr, "pf_groupnorm_train: null descriptor");
  PF_REQUIRE(d->b > 0 && d->c > 0 && d->t > 0 && d->h > 0 && d->w > 0, "pf_groupnorm_train: bad shape");
  PF_REQUIRE(d->groups > 0 && d->c % d->groups == 0, "pf_groupnorm_train: channels=%d is not a multiple of groups=%d", d->c,
             d->groups);
  PF_REQUIRE(d->c % 8 == 0 && d->c <= 2048, "pf_groupnorm_train: channels=%d must be a multiple of 8, at most 2048", d->c);
  PF_REQUIRE(d->x_f32 == 0 || d->x_f32 == 1, "pf_groupnorm_train: x_f32 must be 0 (bf16) or 1 (fp32)");
  PF_REQUIRE(d->silu == 0 || d->silu == 1, "pf_groupnorm_train: silu must be 0 or 1");
  const long long frames = static_cast<long long>(d->b) * d->t;
  PF_REQUIRE(frames < 65536 && frames * d->c < (1ll << 31), "pf_groupnorm_train: too many frames");
  p = GtPlan{};
  GnArgs& a = p.a;
  a.b = d->b; a.c = d->c; a.t = d->t; a.groups = d->groups; a.cpg = d->c / d->groups; a.silu = d->silu; a.eps = d->eps;
  a.voxels = static_cast<long long>(d->h) * d->w;
  a.nsplit = gn_splits(a.voxels);
  PF_REQUIRE(a.voxels * (d->c / 8) / GT_THREADS < (1ll << 31), "pf_groupnorm_train: frame of %lld voxels is too large",
             a.voxels);
  a.x = d->x; a.gamma = d->gamma; a.beta = d->beta; a.stats = d->stats;
  p.x_f32 = d->x_f32;
  p.ws_need = frames * a.nsplit * d->c * 2 + frames * d->groups * 2;
  long long s[5];
  p.form = gt_form(d->x, d->x_strides, d->b, d->c, d->t, d->h, d->w, s);
  PF_REQUIRE(p.form != 0, "pf_groupnorm_train: x strides (%lld, %lld, %lld, %lld, %lld) are neither channels_last_3d nor "
             "unit-stride (h, w) planes", static_cast<long long>(d->x_strides[0]), static_cast<long long>(d->x_strides[1]),
             static_cast<long long>(d->x_strides[2]), static_cast<long long>(d->x_strides[3]),
             static_cast<long long>(d->x_strides[4]));
  for (int i = 0; i < 3; ++i) a.xs[i] = s[i];
  bool aligned = a.voxels % 8 == 0 && s[0] % 8 == 0 && s[1] % 8 == 0 && s[2] % 8 == 0 &&
                 (reinterpret_cast<uintptr_t>(d->x) & 15) == 0;
  if (bwd) {
    PF_REQUIRE(d->dy_f32 == 0 || d->dy_f32 == 1, "pf_groupnorm_train: dy_f32 must be 0 (bf16) or 1 (fp32)");
    long long sd[5];
    const int dform = gt_form(d->dy, d->dy_strides, d->b, d->c, d->t, d->h, d->w, sd);
    PF_REQUIRE(dform == p.form, "pf_groupnorm_train: dy is not in x's layout form (%s)",
               p.form == GT_FORM_CHANNEL ? "channels_last_3d" : "unit-stride (h, w) planes");
    for (int i = 0; i < 3; ++i) a.ds[i] = sd[i];
    aligned = aligned && sd[0] % 8 == 0 && sd[1] % 8 == 0 && sd[2] % 8 == 0 && (reinterpret_cast<uintptr_t>(d->dy) & 15) == 0;
    a.dy = d->dy;
    a.out = d->dx;
    p.t2_f32 = d->dy_f32;
  } else {
    PF_REQUIRE(d->y_f32 == 0 || d->y_f32 == 1, "pf_groupnorm_train: y_f32 must be 0 (bf16) or 1 (fp32)");
    a.dy = d->x;
    for (int i = 0; i < 3; ++i) a.ds[i] = s[i];
    a.out = d->y;
    p.t2_f32 = d->y_f32;
  }
  p.vec = p.form == GT_FORM_PLANE && aligned && (reinterpret_cast<uintptr_t>(a.out) & 15) == 0;
  return 0;
}

static int gt_require_workspace(const pf_groupnorm_train_desc* d, const GtPlan& p, const char* what) {
  PF_REQUIRE(d->workspace != nullptr && d->workspace_floats >= p.ws_need,
             "%s: workspace of %lld floats is too small: this shape needs %lld (pf_groupnorm_train_workspace)", what,
             static_cast<long long>(d->workspace_floats), p.ws_need);
  return 0;
}

static dim3 gt_elem_grid(const GtPlan& p) {
  const GnArgs& a = p.a;
  if (p.form == GT_FORM_CHANNEL)
    return dim3(static_cast<unsigned>((a.voxels * (a.c / 8) + GT_THREADS - 1) / GT_THREADS), a.b * a.t);
  const long long n = p.vec ? a.voxels / 8 : a.voxels;
  const long long chunks = (n + GT_THREADS - 1) / GT_THREADS;
  return dim3(a.b * a.c * a.t, static_cast<unsigned>(chunks < 65535 ? chunks : 65535));
}

template <typename Tx, typename To>
static int gt_forward(const GtPlan& p, float* stats, cudaStream_t st) {
  const GnArgs& a = p.a;
  const int frames = a.b * a.t;
  if (p.form == GT_FORM_CHANNEL) {
    const size_t smem = static_cast<size_t>(GT_THREADS / (a.c / 8)) * a.c * 2 * sizeof(float);
    gt_stats_cl_kernel<Tx><<<frames * a.nsplit, GT_THREADS, smem, st>>>(a);
  } else if (p.vec) {
    gt_partial_pl_kernel<false, true, Tx, Tx><<<frames * a.nsplit, GT_THREADS, 0, st>>>(a);
  } else {
    gt_partial_pl_kernel<false, false, Tx, Tx><<<frames * a.nsplit, GT_THREADS, 0, st>>>(a);
  }
  if (int rc = check_launch("pf_groupnorm_train_fwd (partial sums)")) return rc;
  const int n = frames * a.groups;
  gt_finalize_kernel<Tx><<<(n + 127) / 128, 128, 0, st>>>(a, stats);
  if (int rc = check_launch("pf_groupnorm_train_fwd (finalize)")) return rc;
  const dim3 grid = gt_elem_grid(p);
  if (p.form == GT_FORM_CHANNEL) gt_elem_cl_kernel<false, Tx, Tx, To><<<grid, GT_THREADS, 0, st>>>(a);
  else if (p.vec) gt_elem_pl_kernel<false, true, Tx, Tx, To><<<grid, GT_THREADS, 0, st>>>(a);
  else gt_elem_pl_kernel<false, false, Tx, Tx, To><<<grid, GT_THREADS, 0, st>>>(a);
  return check_launch("pf_groupnorm_train_fwd (apply)");
}

template <typename Tx, typename Td>
static int gt_backward(const GtPlan& p, float* coef, float* dgamma, float* dbeta, cudaStream_t st) {
  GnArgs a = p.a;
  const int frames = a.b * a.t;
  if (p.form == GT_FORM_CHANNEL) {
    const dim3 grid(frames * a.nsplit, (a.c + GT_SLICE - 1) / GT_SLICE);
    gt_bwd_partial_cl_kernel<Tx, Td><<<grid, GT_THREADS, 0, st>>>(a);
  } else if (p.vec) {
    gt_partial_pl_kernel<true, true, Tx, Td><<<frames * a.nsplit, GT_THREADS, 0, st>>>(a);
  } else {
    gt_partial_pl_kernel<true, false, Tx, Td><<<frames * a.nsplit, GT_THREADS, 0, st>>>(a);
  }
  if (int rc = check_launch("pf_groupnorm_train_bwd (partial sums)")) return rc;
  if (dgamma || dbeta) {
    gt_param_grad_kernel<<<(a.c + 127) / 128, 128, 0, st>>>(a, dgamma, dbeta);
    if (int rc = check_launch("pf_groupnorm_train_bwd (dgamma, dbeta)")) return rc;
  }
  if (a.out == nullptr) return 0;
  const int n = frames * a.groups;
  gt_bwd_coef_kernel<<<(n + 127) / 128, 128, 0, st>>>(a, coef);
  if (int rc = check_launch("pf_groupnorm_train_bwd (finalize)")) return rc;
  a.coef = coef;
  const dim3 grid = gt_elem_grid(p);
  if (p.form == GT_FORM_CHANNEL) gt_elem_cl_kernel<true, Tx, Td, Tx><<<grid, GT_THREADS, 0, st>>>(a);
  else if (p.vec) gt_elem_pl_kernel<true, true, Tx, Td, Tx><<<grid, GT_THREADS, 0, st>>>(a);
  else gt_elem_pl_kernel<true, false, Tx, Td, Tx><<<grid, GT_THREADS, 0, st>>>(a);
  return check_launch("pf_groupnorm_train_bwd (dx)");
}

}  // namespace pf

extern "C" int64_t pf_groupnorm_train_workspace(const pf_groupnorm_train_desc* d) {
  pf::GtPlan p;
  if (pf::gt_plan(d, false, p)) return -1;
  return p.ws_need;
}

extern "C" int pf_groupnorm_train_fwd(const pf_groupnorm_train_desc* d, void* stream_) {
  using namespace pf;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  GtPlan p;
  if (int rc = gt_plan(d, false, p)) return rc;
  PF_REQUIRE(d->x && d->gamma && d->beta && d->stats && d->y, "pf_groupnorm_train_fwd: null pointer");
  if (int rc = gt_require_workspace(d, p, "pf_groupnorm_train_fwd")) return rc;
  p.a.partial = d->workspace;
  using bf = __nv_bfloat16;
  if (p.x_f32) return p.t2_f32 ? gt_forward<float, float>(p, d->stats, st) : gt_forward<float, bf>(p, d->stats, st);
  return p.t2_f32 ? gt_forward<bf, float>(p, d->stats, st) : gt_forward<bf, bf>(p, d->stats, st);
}

extern "C" int pf_groupnorm_train_bwd(const pf_groupnorm_train_desc* d, void* stream_) {
  using namespace pf;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  GtPlan p;
  if (int rc = gt_plan(d, true, p)) return rc;
  PF_REQUIRE(d->x && d->dy && d->gamma && d->beta && d->stats, "pf_groupnorm_train_bwd: null pointer");
  if (int rc = gt_require_workspace(d, p, "pf_groupnorm_train_bwd")) return rc;
  p.a.partial = d->workspace;
  float* coef = d->workspace + (p.ws_need - static_cast<long long>(d->b) * d->t * d->groups * 2);
  using bf = __nv_bfloat16;
  if (p.x_f32)
    return p.t2_f32 ? gt_backward<float, float>(p, coef, d->dgamma, d->dbeta, st)
                    : gt_backward<float, bf>(p, coef, d->dgamma, d->dbeta, st);
  return p.t2_f32 ? gt_backward<bf, float>(p, coef, d->dgamma, d->dbeta, st)
                  : gt_backward<bf, bf>(p, coef, d->dgamma, d->dbeta, st);
}
