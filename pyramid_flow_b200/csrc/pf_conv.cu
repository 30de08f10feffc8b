// pf_conv.cu — causal 3-D convolution (k = 3x3x3 or 1x1x1, stride 1) as an im2col-free implicit GEMM on Hopper wgmma.
//
// Replaces CausalConv3d -> nn.Conv3d (reference video_vae/modeling_causal_conv.py:116-146, cuDNN conv3d on NCDHW) for
// the VAE decoder.  Activations are channels-last bf16 [B, T, H, W, C]; an output tile is a TH x TW spatial patch of one
// frame (128 voxels = two 64-row wgmma slices), and the K loop walks (tap, 64-channel chunk):
//   A tile  = ONE 5-D TMA box (64 ch, TW, TH, 1 frame, 1 batch) at the tap-shifted coordinate.  Out-of-bounds spatial
//             coordinates are zero-filled by TMA => the conv's spatial zero padding costs nothing; the causal temporal
//             padding is (kt-1) leading frames physically present in the input buffer (zeros for the first chunk, the
//             previous chunk's last frames afterwards — the reference's feature cache, C:126-143).
//   B tile  = weights re-laid out as [Cout, taps*Cin] (tap-major), a plain 2-D TMA box like the GEMM.
// The box lands in shared memory as [TH][TW][64] = 128 rows of 128 B with SWIZZLE_128B, i.e. exactly the K-major wgmma
// operand; no im2col buffer exists anywhere.  Pipeline / warp roles are the GEMM's (pf_gemm.cu).
// Epilogue: bias (+ residual) -> bf16/fp32 channels-last store, optionally through the depth-to-space addressing of
// CausalUpsample2x (R:616) / CausalTemporalUpsample2x (R:724-727) so the rearrange copy disappears.
#include <cstdlib>

#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

struct ConvArgs {
  int b, t, h, w, cin;
  int cout;            // padded N actually computed (multiple of BN)
  int taps, kt, kh, kw;
  int st, sh, sw;      // conv stride (t, h, w): 1, or 2 for the encoder's down-samplers; (b, t, h, w) are OUTPUT dims
  int th, tw, tiles_h, tiles_w;
  int n_tiles;
  const float* bias;
  int store_mode;      // 0 plain, 1 spatial depth-to-space (c p1 p2), 2 temporal depth-to-space (c p)
  void* out;
  int out_f32;
  int out_t_total, out_t_offset, out_h, out_w, out_c;   // geometry of the output buffer
  int store_channels;  // channels of the conv output that are stored (<= cout; the rest is padding)
  const __nv_bfloat16* residual;   // plain mode only; same geometry as out (bf16)
  int res_t_total, res_t_offset;
};

constexpr int CBK = PIPE_BK;

// Epilogue of one staged accumulator row: this thread owns voxel (bb, tt, hh, ww) and every second 16-channel chunk
// (starting at chunk `half`) of conv channels [n_base, n_base+BN); `srow` = the voxel's fp32 accumulators in shared memory.
template <int BN>
__device__ __forceinline__ void conv_epilogue_tile(const ConvArgs& g, const float* srow, int half, int bb, int tt, int hh,
                                                   int ww, bool valid, int n_base) {
#pragma unroll 1
  for (int c = half; c < BN / 16; c += 2) {
    const int n0 = n_base + c * 16;
    if (!valid || n0 >= g.store_channels) continue;
    float x[16];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float4 v = *reinterpret_cast<const float4*>(srow + c * 16 + 4 * i);
      x[4 * i + 0] = v.x + (g.bias ? __ldg(g.bias + n0 + 4 * i + 0) : 0.f);
      x[4 * i + 1] = v.y + (g.bias ? __ldg(g.bias + n0 + 4 * i + 1) : 0.f);
      x[4 * i + 2] = v.z + (g.bias ? __ldg(g.bias + n0 + 4 * i + 2) : 0.f);
      x[4 * i + 3] = v.w + (g.bias ? __ldg(g.bias + n0 + 4 * i + 3) : 0.f);
    }
    if (g.store_mode == 0) {
      const int to = tt + g.out_t_offset;
      if (to < 0 || to >= g.out_t_total) continue;
      const size_t vox = ((static_cast<size_t>(bb) * g.out_t_total + to) * g.out_h + hh) * g.out_w + ww;
      if (g.residual != nullptr) {
        const size_t rvox = ((static_cast<size_t>(bb) * g.res_t_total + (tt + g.res_t_offset)) * g.out_h + hh) * g.out_w + ww;
        const uint4* r4 = reinterpret_cast<const uint4*>(g.residual + rvox * g.out_c + n0);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const uint4 rv = __ldg(r4 + u);
          const __nv_bfloat162* hv = reinterpret_cast<const __nv_bfloat162*>(&rv);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = __bfloat1622float2(hv[i]);
            x[8 * u + 2 * i] += f.x;
            x[8 * u + 2 * i + 1] += f.y;
          }
        }
      }
      const int nvalid = g.store_channels - n0;
      if (g.out_f32 == 2) {
        // uint8 image store of decode_latent (P:1238): clamp(v * 127.5 + 127.5, 0, 255), truncated like torch's .byte()
        uint8_t* dst = reinterpret_cast<uint8_t*>(g.out) + vox * g.out_c + n0;
#pragma unroll
        for (int i = 0; i < 16; ++i)
          if (i < nvalid) dst[i] = static_cast<uint8_t>(fminf(fmaxf(fmaf(x[i], 127.5f, 127.5f), 0.f), 255.f));
      } else if (g.out_f32) {
        float* dst = reinterpret_cast<float*>(g.out) + vox * g.out_c + n0;
        if (nvalid >= 16 && (g.out_c & 3) == 0) {
#pragma unroll
          for (int i = 0; i < 4; ++i)
            reinterpret_cast<float4*>(dst)[i] = make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
        } else {
#pragma unroll
          for (int i = 0; i < 16; ++i)
            if (i < nvalid) dst[i] = x[i];
        }
      } else {
        __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(g.out) + vox * g.out_c + n0;
        if (nvalid >= 16 && (g.out_c & 7) == 0) {
          uint4 u0, u1;
          u0.x = pack_bf16x2(x[0], x[1]); u0.y = pack_bf16x2(x[2], x[3]); u0.z = pack_bf16x2(x[4], x[5]); u0.w = pack_bf16x2(x[6], x[7]);
          u1.x = pack_bf16x2(x[8], x[9]); u1.y = pack_bf16x2(x[10], x[11]); u1.z = pack_bf16x2(x[12], x[13]); u1.w = pack_bf16x2(x[14], x[15]);
          reinterpret_cast<uint4*>(dst)[0] = u0;
          reinterpret_cast<uint4*>(dst)[1] = u1;
        } else {
#pragma unroll
          for (int i = 0; i < 16; ++i)
            if (i < nvalid) dst[i] = __float2bfloat16(x[i]);
        }
      }
    } else if (g.store_mode == 1) {
      // 'b (c p1 p2) t h w -> b c t (h p1) (w p2)': conv channel n = 4c + 2 p1 + p2; 16 n = 4 output channels x 4 pixels
      const int to = tt + g.out_t_offset;
      if (to < 0 || to >= g.out_t_total) continue;
      const int c0 = n0 >> 2;
      __nv_bfloat16* base = reinterpret_cast<__nv_bfloat16*>(g.out);
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int p1 = p >> 1, p2 = p & 1;
        const size_t vox = ((static_cast<size_t>(bb) * g.out_t_total + to) * g.out_h + (2 * hh + p1)) * g.out_w + (2 * ww + p2);
        uint2 u;
        u.x = pack_bf16x2(x[0 + p], x[4 + p]);
        u.y = pack_bf16x2(x[8 + p], x[12 + p]);
        *reinterpret_cast<uint2*>(base + vox * g.out_c + c0) = u;
      }
    } else {
      // 'b (c p) t h w -> b c (t p) h w': conv channel n = 2c + p; frame 2t + p (+offset; negative = dropped frame)
      const int c0 = n0 >> 1;
      __nv_bfloat16* base = reinterpret_cast<__nv_bfloat16*>(g.out);
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int to = 2 * tt + p + g.out_t_offset;
        if (to < 0 || to >= g.out_t_total) continue;
        const size_t vox = ((static_cast<size_t>(bb) * g.out_t_total + to) * g.out_h + hh) * g.out_w + ww;
        uint4 u;
        u.x = pack_bf16x2(x[0 + p], x[2 + p]);
        u.y = pack_bf16x2(x[4 + p], x[6 + p]);
        u.z = pack_bf16x2(x[8 + p], x[10 + p]);
        u.w = pack_bf16x2(x[12 + p], x[14 + p]);
        *reinterpret_cast<uint4*>(base + vox * g.out_c + c0) = u;
      }
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(PIPE_THREADS, 1)
conv3d_wgmma_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w, const ConvArgs g) {
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
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_w);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], PIPE_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int cchunks = g.cin / CBK;
  const int num_kb = g.taps * cchunks;
  // tile index -> (n tile fastest, then spatial tile, frame, batch): CTAs running together share the same input patch
  const int sp_tiles = g.tiles_h * g.tiles_w;
  const long long total_tiles = static_cast<long long>(g.b) * g.t * sp_tiles * g.n_tiles;

  if (wgroup == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // ===== TMA producer =====
      int stage = 0;
      uint32_t phase = 0;
      const int ph = g.kh >> 1, pw = g.kw >> 1;
      for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = static_cast<int>(tile % g.n_tiles);
        long long r = tile / g.n_tiles;
        const int sp = static_cast<int>(r % sp_tiles);
        r /= sp_tiles;
        const int tt = static_cast<int>(r % g.t);
        const int bb = static_cast<int>(r / g.t);
        const int h0 = (sp / g.tiles_w) * g.th, w0 = (sp % g.tiles_w) * g.tw;
        for (int kb = 0; kb < num_kb; ++kb) {
          // K order (dt, dh, channel chunk, dw)
          const int grp = kb / g.kw;
          const int dw = kb - grp * g.kw;
          const int dtdh = grp / cchunks;
          const int cc = grp - dtdh * cchunks;
          const int dt = dtdh / g.kh, dh = dtdh - dt * g.kh;
          const int wk = (dtdh * g.kw + dw) * cchunks + cc;     // K block of tap (dt, dh, dw), chunk cc in the weight matrix
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          tma_load_5d(sa, &tm_x, &full_bar[stage], cc * CBK, w0 * g.sw + dw - pw, h0 * g.sh + dh - ph, tt * g.st + dt, bb);
          tma_load_2d(sa + Cfg::A_BYTES, &tm_w, &full_bar[stage], wk * CBK, nt * BN);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===== consumers: K loop on the tensor cores, then the epilogue (thread == output voxel x channel-chunk parity) =====
    setmaxnreg_inc<232>();
    const int wg = wgroup - 1;
    const int tid = threadIdx.x & 127;
    const int rrow = wg * 64 + (tid & 63);
    const int lh = rrow / g.tw, lw = rrow - lh * g.tw;
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int nt = static_cast<int>(tile % g.n_tiles);
      long long r = tile / g.n_tiles;
      const int sp = static_cast<int>(r % sp_tiles);
      r /= sp_tiles;
      const int tt = static_cast<int>(r % g.t);
      const int bb = static_cast<int>(r / g.t);
      const int hh = (sp / g.tiles_w) * g.th + lh, ww = (sp % g.tiles_w) * g.tw + lw;
      const bool valid = hh < g.h && ww < g.w;
      pipe_consume_tile<BN>(acc, smem, full_bar, empty_bar, num_kb, wg, stage, phase);
      named_bar_sync(1 + wg, 128);   // the previous tile's epilogue reads of this warpgroup's staging rows are done
      pipe_stage_acc<BN>(acc, acc_tile, wg);
      named_bar_sync(1 + wg, 128);
      conv_epilogue_tile<BN>(g, acc_tile + rrow * Cfg::ACC_PITCH, tid >> 6, bb, tt, hh, ww, valid, nt * BN);
    }
  }
}

template <int BN>
static int launch_conv(const CUtensorMap& tm_x, const CUtensorMap& tm_w, const ConvArgs& g, cudaStream_t stream) {
  using Cfg = PipeCfg<BN>;
  auto kern = conv3d_wgmma_kernel<BN>;
  if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(kern), Cfg::SMEM_BYTES, "conv")) return rc;
  const long long total = static_cast<long long>(g.b) * g.t * g.tiles_h * g.tiles_w * g.n_tiles;
  int grid = num_sms();
  if (grid <= 0) grid = 132;
  if (total < grid) grid = static_cast<int>(total);
  kern<<<grid, PIPE_THREADS, Cfg::SMEM_BYTES, stream>>>(tm_x, tm_w, g);
  return check_launch("pf_causal_conv3d");
}

int warmup_conv() {
  int rc = ensure_dyn_smem(reinterpret_cast<const void*>(conv3d_wgmma_kernel<128>), PipeCfg<128>::SMEM_BYTES, "conv<128>");
  if (!rc) rc = ensure_dyn_smem(reinterpret_cast<const void*>(conv3d_wgmma_kernel<64>), PipeCfg<64>::SMEM_BYTES, "conv<64>");
  return rc;
}

}  // namespace pf

extern "C" int pf_causal_conv3d(const pf_conv3d_desc* d, void* stream_) {
  using namespace pf;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  PF_REQUIRE(d && d->x && d->wgt && d->out, "pf_causal_conv3d: null pointer");
  PF_REQUIRE(d->cin % 64 == 0 && d->cin > 0, "pf_causal_conv3d: cin=%d must be a multiple of 64 (pad the channels)", d->cin);
  PF_REQUIRE(d->cout % 64 == 0 && d->cout > 0, "pf_causal_conv3d: cout=%d must be a multiple of 64 (pad the filters)", d->cout);
  PF_REQUIRE((d->kt == 1 || d->kt == 3) && (d->kh == 1 || d->kh == 3) && d->kw == d->kh, "pf_causal_conv3d: kernel must be 1x1x1 or 3x3x3 (kt in {1,3})");
  PF_REQUIRE(d->b > 0 && d->t > 0 && d->h > 0 && d->w > 0, "pf_causal_conv3d: bad shape");
  PF_REQUIRE(d->store_mode >= 0 && d->store_mode <= 2, "pf_causal_conv3d: bad store_mode");
  PF_REQUIRE(d->store_channels > 0 && d->store_channels <= d->cout, "pf_causal_conv3d: bad store_channels");
  if (d->store_mode == 1) PF_REQUIRE(d->store_channels == d->cout && d->out_c * 4 == d->cout && !d->out_f32 && !d->residual, "pf_causal_conv3d: spatial depth-to-space needs out_c = cout/4, bf16, no residual");
  if (d->store_mode == 2) PF_REQUIRE(d->store_channels == d->cout && d->out_c * 2 == d->cout && !d->out_f32 && !d->residual, "pf_causal_conv3d: temporal depth-to-space needs out_c = cout/2, bf16, no residual");
  if (d->store_mode == 0) PF_REQUIRE(d->out_c >= d->store_channels, "pf_causal_conv3d: out_c < store_channels");
  PF_REQUIRE(d->out_f32 >= 0 && d->out_f32 <= 2 && (d->out_f32 != 2 || !d->residual), "pf_causal_conv3d: out_f32 must be 0 (bf16), 1 (fp32) or 2 (uint8 image, no residual)");
  const int st = d->stride_t > 1 ? d->stride_t : 1, sh = d->stride_h > 1 ? d->stride_h : 1, sw = d->stride_w > 1 ? d->stride_w : 1;
  PF_REQUIRE(st <= 2 && sh <= 2 && sw <= 2 && sh == sw, "pf_causal_conv3d: strides must be 1 or 2 with stride_h == stride_w");
  if (st > 1 || sh > 1) PF_REQUIRE(d->store_mode == 0 && d->kt == 3 && d->kh == 3, "pf_causal_conv3d: strided convs are plain-store 3x3x3 (CausalDownsample2x R:322, CausalTemporalDownsample2x R:486)");

  ConvArgs g{};
  g.b = d->b; g.t = d->t; g.h = d->h; g.w = d->w; g.cin = d->cin; g.cout = d->cout;
  g.kt = d->kt; g.kh = d->kh; g.kw = d->kw; g.taps = d->kt * d->kh * d->kw;
  g.st = st; g.sh = sh; g.sw = sw;
  int tw = 128;
  while (tw > 8 && tw / 2 >= d->w) tw >>= 1;   // smallest power of two >= w, clamped to [8, 128]
  g.tw = tw; g.th = 128 / tw;
  g.tiles_w = (d->w + g.tw - 1) / g.tw;
  g.tiles_h = (d->h + g.th - 1) / g.th;
  int bn = (d->cout % 128 == 0) ? 128 : 64;
  g.bias = d->bias;
  g.store_mode = d->store_mode;
  g.out = d->out; g.out_f32 = d->out_f32;
  g.out_t_total = d->out_t_total; g.out_t_offset = d->out_t_offset;
  g.out_h = d->store_mode == 1 ? 2 * d->h : d->h;
  g.out_w = d->store_mode == 1 ? 2 * d->w : d->w;
  g.out_c = d->out_c;
  g.store_channels = d->store_channels;
  g.residual = static_cast<const __nv_bfloat16*>(d->residual);
  g.res_t_total = d->res_t_total; g.res_t_offset = d->res_t_offset;

  // kernel_variant 1 / 2 pins the 128-wide / 64-wide filter tile (same K order, same bits)
  PF_REQUIRE(d->kernel_variant >= 0 && d->kernel_variant <= 2, "pf_causal_conv3d: bad kernel_variant %d", d->kernel_variant);
  PF_REQUIRE(d->kernel_variant != 1 || bn == 128, "pf_causal_conv3d: kernel_variant 1 (128-wide filter tiles) needs cout %% 128 == 0");
  if (d->kernel_variant == 2) bn = 64;
  g.n_tiles = d->cout / bn;
  // input geometry: (t-1)*st + kt frames (the kt-1 causal frames physically first), h*sh x w*sw voxels (symmetric pad 1 is
  // the TMA's out-of-bounds zero fill).  A strided conv loads every sh-th / sw-th voxel of a (th*sh) x (tw*sw) box.
  const int tin = (d->t - 1) * st + d->kt;
  const int hin = d->h * sh, win = d->w * sw;
  CUtensorMap tm_x, tm_w;
  {
    const uint64_t dims[5] = {static_cast<uint64_t>(d->cin), static_cast<uint64_t>(win), static_cast<uint64_t>(hin),
                              static_cast<uint64_t>(tin), static_cast<uint64_t>(d->b)};
    const uint64_t s0 = static_cast<uint64_t>(d->cin) * 2;
    const uint64_t strides[4] = {s0, s0 * win, s0 * win * hin, s0 * win * hin * tin};
    const uint32_t box[5] = {CBK, static_cast<uint32_t>(g.tw * sw), static_cast<uint32_t>(g.th * sh), 1, 1};
    const uint32_t estr[5] = {1, static_cast<uint32_t>(sw), static_cast<uint32_t>(sh), 1, 1};
    int rc = encode_tensor_map(&tm_x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, d->x, dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B, estr);
    if (rc) return rc;
  }
  {
    const uint64_t kdim = static_cast<uint64_t>(g.taps) * d->cin;
    const uint64_t dims[2] = {kdim, static_cast<uint64_t>(d->cout)};
    const uint64_t strides[1] = {kdim * 2};
    const uint32_t box[2] = {CBK, static_cast<uint32_t>(bn)};
    int rc = encode_tensor_map(&tm_w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, d->wgt, dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  if (bn == 128) return launch_conv<128>(tm_x, tm_w, g, stream);
  return launch_conv<64>(tm_x, tm_w, g, stream);
}
