// pf_conv_bwd.cu — backward of the causal 3-D convolution (training of the VAE): activation packing with the bias gradient,
// and the weight gradient as an MN-major wgmma GEMM with a fixed split of the voxel range.
//
// Replaces the autograd of CausalConv3d.forward (reference video_vae/modeling_causal_conv.py:116-126, temporal_chunk=False:
// F.pad(x, (1, 1, 1, 1, 2, 0)) -> nn.Conv3d(padding=0)), i.e. cuDNN's conv3d data / weight / bias gradients.
//
//   pack   : [B, C, T, H, W] (bf16 or fp32, any strides) -> channels-last bf16 [B, T_total, H*dh, W*dw, Cpad]; source voxel
//            (t, h, w) lands at (t_offset + t*dt, h*dh, w*dw), everything else (causal frames, inserted zeros, channel padding)
//            is written as zero.  One CTA per destination row; a 64-channel x 64-voxel tile is transposed through shared
//            memory, loaded 16 / 32 B at a time along W (NCDHW) or C (channels-last) where the strides allow.  With a bias
//            gradient requested, each source row also writes its per-channel sums (fp32, fixed order), and two reduce
//            passes (row groups, then the groups) add them up in an order fixed by the shape.
//   wgrad  : dW[co, tap, ci] = sum over output voxels v of dy[v, co] * x_pad[v*stride + tap, ci] -- M = Cout, N = taps*Cin,
//            K = voxels.  A K block is one 128-voxel tile (TH x TW of one frame); the producer loads, per stage, up to two
//            64-channel dy boxes and two 64-channel x boxes at the tap-shifted coordinate with the forward's element
//            strides, so every box lands as [128 voxel rows][64 channels] with SWIZZLE_128B: the channels (M for dy, N for
//            x) are contiguous, and both operands are MN-major (transposed) wgmma operands.  A CTA owns one (128 co, tap,
//            128 ci) tile and one fixed share of the voxel tiles; the split count depends only on the shape, each split
//            writes its fp32 partial tile to a workspace, and the reduce sums the splits in order into PyTorch's
//            [Cout, Cin, kt, kh, kw] layout.  No atomics: the bits depend on the shape alone.
#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

// ------------------------------------------------------------------------------------------------------------------ pack
constexpr int PK_THREADS = 256;
constexpr int PK_W = 64;   // source voxels per tile
constexpr int PK_C = 64;   // channels per tile
constexpr int PK_VEC = 8;  // elements per vector load
constexpr int BG_GROUPS = 128;  // row groups of the bias gradient's first reduce stage (at most)

struct PackArgs {
  const void* src;
  int src_f32;
  int b, c, t, h, w;
  long long s[5];
  int vec;               // 0: scalar loads; 1: 8 consecutive w per load (w stride 1); 2: 8 consecutive channels (c stride 1)
  int c_fast;            // scalar loads walk channels first (the channel stride is 1)
  __nv_bfloat16* dst;
  int cpad, t_total, t_offset, dt, dh, dw;
  float* partial;        // [b * t * h][cpad] or NULL
};

__device__ __forceinline__ float pack_load(const PackArgs& a, long long off) {
  return a.src_f32 ? __ldg(reinterpret_cast<const float*>(a.src) + off)
                   : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a.src)[off]);
}
// 8 consecutive elements at element offset `off` (a multiple of 8; the host checked the alignment)
__device__ __forceinline__ void pack_load8(const PackArgs& a, long long off, float (&v)[PK_VEC]) {
  if (a.src_f32) {
    const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.src) + off);
    const float4 u0 = __ldg(p), u1 = __ldg(p + 1);
    v[0] = u0.x; v[1] = u0.y; v[2] = u0.z; v[3] = u0.w; v[4] = u1.x; v[5] = u1.y; v[6] = u1.z; v[7] = u1.w;
  } else {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(a.src) + off));
    const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = __bfloat1622float2(h2[k]);
      v[2 * k] = f.x;
      v[2 * k + 1] = f.y;
    }
  }
}

__global__ void __launch_bounds__(PK_THREADS, 4) conv_pack_kernel(const PackArgs a) {
  __shared__ float tile[PK_C][PK_W + 1];
  const int tid = threadIdx.x;
  const int hd = a.h * a.dh, wd = a.w * a.dw;
  const int row = blockIdx.x;
  const int hq = row % hd;
  const int r = row / hd;
  const int tq = r % a.t_total;
  const int bb = r / a.t_total;
  __nv_bfloat16* drow = a.dst + static_cast<size_t>(row) * wd * a.cpad;
  const int ts = tq - a.t_offset;
  const bool valid = ts >= 0 && ts % a.dt == 0 && ts / a.dt < a.t && hq % a.dh == 0;
  if (!valid) {
    uint4* d4 = reinterpret_cast<uint4*>(drow);
    const int n = wd * a.cpad / 8;
    for (int i = tid; i < n; i += PK_THREADS) d4[i] = make_uint4(0, 0, 0, 0);
    return;
  }
  const int ti = ts / a.dt, hi = hq / a.dh;
  const long long base = bb * a.s[0] + ti * a.s[2] + hi * a.s[3];
  for (int cc = 0; cc < a.cpad / PK_C; ++cc) {
    float colsum = 0.f;
    for (int w0 = 0; w0 < a.w; w0 += PK_W) {
      if (a.vec == 1) {
        // [64 channels][8 groups of 8 w]: a warp reads 4 channels x 128 contiguous bytes (bf16) per load
        for (int i = tid; i < PK_C * (PK_W / PK_VEC); i += PK_THREADS) {
          const int cl = i / (PK_W / PK_VEC), wl = (i % (PK_W / PK_VEC)) * PK_VEC;
          const int ch = cc * PK_C + cl, wi = w0 + wl;
          float v[PK_VEC];
          if (ch < a.c && wi + PK_VEC <= a.w) {
            pack_load8(a, base + ch * a.s[1] + wi, v);
          } else {
#pragma unroll
            for (int k = 0; k < PK_VEC; ++k) v[k] = (ch < a.c && wi + k < a.w) ? pack_load(a, base + ch * a.s[1] + wi + k) : 0.f;
          }
#pragma unroll
          for (int k = 0; k < PK_VEC; ++k) tile[cl][wl + k] = v[k];
        }
      } else if (a.vec == 2) {
        // [64 w][8 groups of 8 channels]: channels-last sources
        for (int i = tid; i < PK_W * (PK_C / PK_VEC); i += PK_THREADS) {
          const int wl = i / (PK_C / PK_VEC), cl = (i % (PK_C / PK_VEC)) * PK_VEC;
          const int ch = cc * PK_C + cl, wi = w0 + wl;
          float v[PK_VEC];
          if (wi < a.w && ch + PK_VEC <= a.c) {
            pack_load8(a, base + ch + wi * a.s[4], v);
          } else {
#pragma unroll
            for (int k = 0; k < PK_VEC; ++k) v[k] = (wi < a.w && ch + k < a.c) ? pack_load(a, base + (ch + k) + wi * a.s[4]) : 0.f;
          }
#pragma unroll
          for (int k = 0; k < PK_VEC; ++k) tile[cl + k][wl] = v[k];
        }
      } else {
        for (int i = tid; i < PK_C * PK_W; i += PK_THREADS) {
          const int cl = a.c_fast ? (i % PK_C) : (i / PK_W);
          const int wl = a.c_fast ? (i / PK_C) : (i % PK_W);
          const int ch = cc * PK_C + cl, wi = w0 + wl;
          tile[cl][wl] = (ch < a.c && wi < a.w) ? pack_load(a, base + ch * a.s[1] + wi * a.s[4]) : 0.f;
        }
      }
      __syncthreads();
      if (a.partial != nullptr && tid < PK_C) {
#pragma unroll 8
        for (int j = 0; j < PK_W; ++j) colsum += tile[tid][j];
      }
      const int dv0 = w0 * a.dw;
      const int nv = min(PK_W * a.dw, wd - dv0);
      for (int i = tid; i < nv * (PK_C / 8); i += PK_THREADS) {
        const int vl = i >> 3, q = i & 7;
        const bool here = vl % a.dw == 0;   // else an inserted zero voxel
        const float* col = &tile[q * 8][vl / a.dw];
        uint32_t u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
          u[k] = here ? pack_bf16x2(col[(2 * k) * (PK_W + 1)], col[(2 * k + 1) * (PK_W + 1)]) : 0u;
        *reinterpret_cast<uint4*>(drow + static_cast<size_t>(dv0 + vl) * a.cpad + cc * PK_C + q * 8) = make_uint4(u[0], u[1], u[2], u[3]);
      }
      __syncthreads();
    }
    if (a.partial != nullptr && tid < PK_C)
      a.partial[(static_cast<size_t>(bb * a.t + ti) * a.h + hi) * a.cpad + cc * PK_C + tid] = colsum;
  }
}

// out[g][ch] = sum of partial[row][ch] over the rows of group g (rows [g*rows/G, (g+1)*rows/G), G = gridDim.y); warp k adds
// the group's rows k, k + 8, ..., and the 8 warp sums are added in warp order.  Run with G groups into a [G][cpad] buffer,
// then once more with one group over that buffer: the bias gradient, in an order fixed by the shape.
__global__ void __launch_bounds__(256) conv_bias_grad_kernel(const float* partial, long long rows, int cpad, int c, float* out) {
  __shared__ float part[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ch = blockIdx.x * 32 + lane;
  const long long r0 = blockIdx.y * rows / gridDim.y, r1 = (blockIdx.y + 1) * rows / gridDim.y;
  float s = 0.f;
  for (long long r = r0 + warp; r < r1; r += 8) s += partial[r * cpad + ch];
  part[warp][lane] = s;
  __syncthreads();
  if (warp == 0) {
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) tot += part[k][lane];
    if (gridDim.y > 1) out[static_cast<long long>(blockIdx.y) * cpad + ch] = tot;
    else if (ch < c) out[ch] = tot;
  }
}

// ------------------------------------------------------------------------------------------------------------------ wgrad
constexpr int WG_BOX_BYTES = PIPE_BM * PIPE_BK * 2;      // one [128 voxels][64 channels] bf16 box
constexpr int WG_STAGE_BYTES = 4 * WG_BOX_BYTES;         // dy boxes 0, 1 then x boxes 0, 1
constexpr int WG_STAGES = 3;
constexpr int WG_SMEM_BYTES = WG_STAGES * WG_STAGE_BYTES + 1024;
constexpr int WG_TARGET_CTAS = 2 * 132;                  // about two waves of an H100 SXM; fixed, so the split is shape-only
constexpr long long WG_MAX_WORKSPACE_FLOATS = 1ll << 26; // 256 MiB of split partials at most

struct WgradArgs {
  int b, t, h, w;
  int cin, cout, taps, kh, kw;
  int st, sh, sw;
  int th, tw, tiles_h, tiles_w;
  long long vox_tiles;
  int m_tiles, n_tiles, out_tiles, splits;
  float* ws;
};

// D[64 x 128] (+)= A[smem, MN-major] * B[smem, MN-major] (both operands transposed: M resp. N contiguous)
__device__ __forceinline__ void wgmma_ss_n128_tt(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

__global__ void __launch_bounds__(PIPE_THREADS, 1)
conv3d_wgrad_kernel(const __grid_constant__ CUtensorMap tm_dy, const __grid_constant__ CUtensorMap tm_x, const WgradArgs g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full_bar[WG_STAGES];
  __shared__ __align__(8) uint64_t empty_bar[WG_STAGES];

  const int warp = threadIdx.x >> 5;
  const int wgroup = warp >> 2;
  // work item -> (output tile fastest, then split): CTAs that run together read the same voxel range
  const int ot = blockIdx.x % g.out_tiles;
  const int split = blockIdx.x / g.out_tiles;
  const int nt = ot % g.n_tiles;
  const int tap = (ot / g.n_tiles) % g.taps;
  const int mt = ot / (g.n_tiles * g.taps);
  const int m_boxes = min(2, g.cout / PIPE_BK - 2 * mt);   // 64-channel dy boxes this tile has (the rest is not loaded)
  const int n_boxes = min(2, g.cin / PIPE_BK - 2 * nt);
  const long long v0 = split * g.vox_tiles / g.splits, v1 = (split + 1) * g.vox_tiles / g.splits;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_dy);
    tma_prefetch_desc(&tm_x);
    for (int i = 0; i < WG_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4 * m_boxes);   // one arrival per warp of each warpgroup that has a dy box
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int sp_tiles = g.tiles_h * g.tiles_w;
  if (wgroup == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // ===== TMA producer =====
      const int dt = tap / (g.kh * g.kw), dh = (tap / g.kw) % g.kh, dw = tap % g.kw;
      const int ph = g.kh >> 1, pw = g.kw >> 1;
      int stage = 0;
      uint32_t phase = 0;
      for (long long v = v0; v < v1; ++v) {
        const int sp = static_cast<int>(v % sp_tiles);
        const long long r = v / sp_tiles;
        const int tt = static_cast<int>(r % g.t);
        const int bb = static_cast<int>(r / g.t);
        const int h0 = (sp / g.tiles_w) * g.th, w0 = (sp % g.tiles_w) * g.tw;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* s = smem + stage * WG_STAGE_BYTES;
        mbar_arrive_expect_tx(&full_bar[stage], (m_boxes + n_boxes) * WG_BOX_BYTES);
        for (int j = 0; j < m_boxes; ++j)
          tma_load_5d(s + j * WG_BOX_BYTES, &tm_dy, &full_bar[stage], (2 * mt + j) * PIPE_BK, w0 * g.sw, h0 * g.sh,
                      tt * g.st, bb);
        for (int j = 0; j < n_boxes; ++j)
          tma_load_5d(s + (2 + j) * WG_BOX_BYTES, &tm_x, &full_bar[stage], (2 * nt + j) * PIPE_BK, w0 * g.sw + dw - pw,
                      h0 * g.sh + dh - ph, tt * g.st + dt, bb);
        if (++stage == WG_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // ===== consumers: warpgroup wg owns output channels [128 mt + 64 wg, +64) x the 128 input channels of the tile =====
    setmaxnreg_inc<232>();
    const int wg = wgroup - 1;
    if (wg >= m_boxes) return;
    const int lane = threadIdx.x & 31;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (long long v = v0; v < v1; ++v) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t s = smem_u32(smem + stage * WG_STAGE_BYTES);
      // MN-major SWIZZLE_128B: 8 voxel rows of 128 B per 1024 B atom (SBO), a 16-voxel K step = +2048 B; the second
      // 64-channel x box is the next MN atom, 16 KiB on (LBO).
      const uint64_t da = make_smem_desc(s + wg * WG_BOX_BYTES, WG_BOX_BYTES, 1024);
      const uint64_t db = make_smem_desc(s + 2 * WG_BOX_BYTES, WG_BOX_BYTES, 1024);
      wgmma_reg_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < PIPE_BM / 16; ++kk) wgmma_ss_n128_tt(acc, da + 128 * kk, db + 128 * kk, 1u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == WG_STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_reg_fence(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    // fragments -> workspace [split][cout][taps][cin] (columns of a missing second x box are dropped)
    const int w4 = warp & 3;
    const int co = 128 * mt + 64 * wg + 16 * w4 + (lane >> 2);
    const long long ld = static_cast<long long>(g.taps) * g.cin;
    float* r0 = g.ws + (static_cast<long long>(split) * g.cout + co) * ld + static_cast<long long>(tap) * g.cin + 128 * nt +
                2 * (lane & 3);
    float* r1 = r0 + 8 * ld;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      if (i < 8 * n_boxes) {
        *reinterpret_cast<float2*>(r0 + 8 * i) = make_float2(acc[4 * i + 0], acc[4 * i + 1]);
        *reinterpret_cast<float2*>(r1 + 8 * i) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
      }
    }
  }
}

// dw[co, ci, tap] = sum over splits s (in order) of ws[s][co][tap][ci], for co < cout_real, ci < cin_real
__global__ void __launch_bounds__(256) conv_wgrad_reduce_kernel(const float* ws, int splits, int cout, int cin, int taps,
                                                                int cout_real, int cin_real, float* dw) {
  const long long n = static_cast<long long>(cout_real) * taps * cin;
  const long long stride = static_cast<long long>(cout) * taps * cin;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    const int ci = static_cast<int>(i % cin);
    if (ci >= cin_real) continue;
    const long long r = i / cin;
    const int tap = static_cast<int>(r % taps);
    const int co = static_cast<int>(r / taps);
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += ws[k * stride + i];
    dw[(static_cast<long long>(co) * cin_real + ci) * taps + tap] = s;
  }
}

static int wgrad_plan(const pf_conv3d_wgrad_desc* d, WgradArgs& g) {
  PF_REQUIRE(d != nullptr, "pf_conv3d_wgrad: null descriptor");
  PF_REQUIRE(d->cin % 64 == 0 && d->cin > 0 && d->cout % 64 == 0 && d->cout > 0,
             "pf_conv3d_wgrad: cin=%d / cout=%d must be positive multiples of 64 (pad the channels)", d->cin, d->cout);
  PF_REQUIRE(d->cin_real > 0 && d->cin_real <= d->cin && d->cout_real > 0 && d->cout_real <= d->cout,
             "pf_conv3d_wgrad: bad cin_real / cout_real");
  PF_REQUIRE((d->kt == 1 || d->kt == 3) && (d->kh == 1 || d->kh == 3) && d->kw == d->kh,
             "pf_conv3d_wgrad: kernel must be 1x1x1 or 3x3x3 (kt in {1,3})");
  PF_REQUIRE(d->b > 0 && d->t > 0 && d->h > 0 && d->w > 0, "pf_conv3d_wgrad: bad shape");
  const int st = d->stride_t > 1 ? d->stride_t : 1, sh = d->stride_h > 1 ? d->stride_h : 1, sw = d->stride_w > 1 ? d->stride_w : 1;
  PF_REQUIRE(st <= 2 && sh <= 2 && sw <= 2 && sh == sw, "pf_conv3d_wgrad: strides must be 1 or 2 with stride_h == stride_w");
  if (st > 1 || sh > 1) PF_REQUIRE(d->kt == 3 && d->kh == 3, "pf_conv3d_wgrad: strided convs are 3x3x3");
  PF_REQUIRE(d->dy_t_total >= (d->t - 1) * st + 1, "pf_conv3d_wgrad: dy_t_total=%d < the %d frames the output covers",
             d->dy_t_total, (d->t - 1) * st + 1);
  g = WgradArgs{};
  g.b = d->b; g.t = d->t; g.h = d->h; g.w = d->w;
  g.cin = d->cin; g.cout = d->cout; g.kh = d->kh; g.kw = d->kw; g.taps = d->kt * d->kh * d->kw;
  g.st = st; g.sh = sh; g.sw = sw;
  int tw = 128;
  while (tw > 8 && tw / 2 >= d->w) tw >>= 1;   // the forward's tile: smallest power of two >= w, clamped to [8, 128]
  g.tw = tw; g.th = 128 / tw;
  g.tiles_w = (d->w + g.tw - 1) / g.tw;
  g.tiles_h = (d->h + g.th - 1) / g.th;
  g.vox_tiles = static_cast<long long>(d->b) * d->t * g.tiles_h * g.tiles_w;
  g.m_tiles = (d->cout / 64 + 1) / 2;
  g.n_tiles = (d->cin / 64 + 1) / 2;
  g.out_tiles = g.m_tiles * g.taps * g.n_tiles;
  const long long out_floats = static_cast<long long>(d->cout) * g.taps * d->cin;
  long long splits = WG_TARGET_CTAS / g.out_tiles;
  if (splits > WG_MAX_WORKSPACE_FLOATS / out_floats) splits = WG_MAX_WORKSPACE_FLOATS / out_floats;
  if (splits > g.vox_tiles) splits = g.vox_tiles;
  if (splits < 1) splits = 1;
  g.splits = static_cast<int>(splits);
  return 0;
}

int warmup_conv_bwd() {
  return ensure_dyn_smem(reinterpret_cast<const void*>(conv3d_wgrad_kernel), WG_SMEM_BYTES, "conv_wgrad");
}

}  // namespace pf

extern "C" int pf_conv3d_pack(const pf_conv3d_pack_desc* d, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(d && d->src && d->dst, "pf_conv3d_pack: null pointer");
  PF_REQUIRE(d->b > 0 && d->c > 0 && d->t > 0 && d->h > 0 && d->w > 0, "pf_conv3d_pack: bad shape");
  PF_REQUIRE(d->cpad % 64 == 0 && d->cpad >= d->c, "pf_conv3d_pack: cpad=%d must be a multiple of 64 and >= c=%d", d->cpad, d->c);
  PF_REQUIRE(d->dil_t >= 1 && d->dil_h >= 1 && d->dil_w >= 1 && d->dil_t <= 2 && d->dil_h <= 2 && d->dil_w <= 2,
             "pf_conv3d_pack: dilations must be 1 or 2");
  PF_REQUIRE(d->t_offset >= 0 && d->t_offset + (d->t - 1) * d->dil_t < d->t_total,
             "pf_conv3d_pack: t_total=%d cannot hold %d frames at offset %d", d->t_total, d->t, d->t_offset);
  PF_REQUIRE(d->src_f32 == 0 || d->src_f32 == 1, "pf_conv3d_pack: src_f32 must be 0 (bf16) or 1 (fp32)");
  const long long rows = static_cast<long long>(d->b) * d->t * d->h;
  const int groups = static_cast<int>(rows < BG_GROUPS ? rows : BG_GROUPS);
  if (d->bias_grad) {
    const long long need = (rows + groups) * d->cpad;
    PF_REQUIRE(d->workspace != nullptr && d->workspace_floats >= need,
               "pf_conv3d_pack: the bias gradient needs a workspace of %lld floats (got %lld)", need,
               static_cast<long long>(d->workspace_floats));
  }
  const long long grid = static_cast<long long>(d->b) * d->t_total * d->h * d->dil_h;
  PF_REQUIRE(grid < (1ll << 31), "pf_conv3d_pack: too many rows");
  PackArgs a{};
  a.src = d->src; a.src_f32 = d->src_f32;
  a.b = d->b; a.c = d->c; a.t = d->t; a.h = d->h; a.w = d->w;
  for (int i = 0; i < 5; ++i) a.s[i] = d->strides[i];
  a.c_fast = d->strides[1] == 1 && d->c > 1;
  // vector loads: 8 consecutive elements along the unit-stride axis, every other stride a multiple of 8 and the base
  // 16-byte aligned, so each vector starts on a 16-byte (bf16) / 32-byte (fp32) boundary
  bool aligned = (reinterpret_cast<uintptr_t>(d->src) & 15) == 0;
  const bool w_unit = d->strides[4] == 1, c_unit = d->strides[1] == 1 && d->c > 1;
  for (int i = 0; i < 5; ++i)
    if (!((i == 4 && w_unit) || (i == 1 && c_unit && !w_unit)) && d->strides[i] % PK_VEC != 0) aligned = false;
  a.vec = !aligned ? 0 : (w_unit ? 1 : (c_unit ? 2 : 0));
  a.dst = static_cast<__nv_bfloat16*>(d->dst);
  a.cpad = d->cpad; a.t_total = d->t_total; a.t_offset = d->t_offset;
  a.dt = d->dil_t; a.dh = d->dil_h; a.dw = d->dil_w;
  a.partial = d->bias_grad ? d->workspace : nullptr;
  conv_pack_kernel<<<static_cast<int>(grid), PK_THREADS, 0, stream>>>(a);
  if (int rc = check_launch("pf_conv3d_pack")) return rc;
  if (!d->bias_grad) return 0;
  float* grouped = d->workspace + rows * d->cpad;
  conv_bias_grad_kernel<<<dim3(d->cpad / 32, groups), 256, 0, stream>>>(d->workspace, rows, d->cpad, d->c, grouped);
  if (int rc = check_launch("pf_conv3d_pack (bias gradient, row groups)")) return rc;
  conv_bias_grad_kernel<<<d->cpad / 32, 256, 0, stream>>>(grouped, groups, d->cpad, d->c, d->bias_grad);
  return check_launch("pf_conv3d_pack (bias gradient)");
}

extern "C" int64_t pf_conv3d_wgrad_workspace(const pf_conv3d_wgrad_desc* d) {
  pf::WgradArgs g;
  if (pf::wgrad_plan(d, g)) return -1;
  return static_cast<int64_t>(g.splits) * d->cout * g.taps * d->cin;
}

extern "C" int pf_conv3d_wgrad(const pf_conv3d_wgrad_desc* d, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  WgradArgs g;
  if (int rc = wgrad_plan(d, g)) return rc;
  PF_REQUIRE(d->x && d->dy && d->dw, "pf_conv3d_wgrad: null pointer");
  const long long need = static_cast<long long>(g.splits) * d->cout * g.taps * d->cin;
  PF_REQUIRE(d->workspace != nullptr && d->workspace_floats >= need,
             "pf_conv3d_wgrad: workspace of %lld floats is too small: this shape needs %lld (pf_conv3d_wgrad_workspace)",
             static_cast<long long>(d->workspace_floats), need);
  g.ws = d->workspace;
  const int tin = (d->t - 1) * g.st + d->kt;
  const int hin = d->h * g.sh, win = d->w * g.sw;
  CUtensorMap tm_dy, tm_x;
  const uint32_t box[5] = {PIPE_BK, static_cast<uint32_t>(g.tw * g.sw), static_cast<uint32_t>(g.th * g.sh), 1, 1};
  const uint32_t estr[5] = {1, static_cast<uint32_t>(g.sw), static_cast<uint32_t>(g.sh), 1, 1};
  {
    const uint64_t dims[5] = {static_cast<uint64_t>(d->cout), static_cast<uint64_t>(win), static_cast<uint64_t>(hin),
                              static_cast<uint64_t>(d->dy_t_total), static_cast<uint64_t>(d->b)};
    const uint64_t s0 = static_cast<uint64_t>(d->cout) * 2;
    const uint64_t strides[4] = {s0, s0 * win, s0 * win * hin, s0 * win * hin * d->dy_t_total};
    if (int rc = encode_tensor_map(&tm_dy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, d->dy, dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B, estr))
      return rc;
  }
  {
    const uint64_t dims[5] = {static_cast<uint64_t>(d->cin), static_cast<uint64_t>(win), static_cast<uint64_t>(hin),
                              static_cast<uint64_t>(tin), static_cast<uint64_t>(d->b)};
    const uint64_t s0 = static_cast<uint64_t>(d->cin) * 2;
    const uint64_t strides[4] = {s0, s0 * win, s0 * win * hin, s0 * win * hin * tin};
    if (int rc = encode_tensor_map(&tm_x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, d->x, dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B, estr))
      return rc;
  }
  if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(conv3d_wgrad_kernel), WG_SMEM_BYTES, "conv_wgrad")) return rc;
  conv3d_wgrad_kernel<<<g.out_tiles * g.splits, PIPE_THREADS, WG_SMEM_BYTES, stream>>>(tm_dy, tm_x, g);
  if (int rc = check_launch("pf_conv3d_wgrad")) return rc;
  const long long n = static_cast<long long>(d->cout_real) * g.taps * d->cin;
  const int blocks = static_cast<int>(n / 256 + 1 < 4096 ? n / 256 + 1 : 4096);
  conv_wgrad_reduce_kernel<<<blocks, 256, 0, stream>>>(d->workspace, g.splits, d->cout, d->cin, g.taps, d->cout_real,
                                                       d->cin_real, d->dw);
  return check_launch("pf_conv3d_wgrad (split reduce)");
}
