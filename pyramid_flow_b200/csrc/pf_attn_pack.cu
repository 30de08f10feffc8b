// pf_attn_pack.cu — the head-major q / k / v of the masked attention's training path, with the reference's RoPE, and the
// backward: per stage (pf_attn_stage_pack), or every stage of a call site packed without its padded rows (pf_attn_varlen_pack,
// with the output scatter pf_attn_varlen_unpack).
//
// Memory-bound: every source element is read once and every packed element written once.  A thread owns 8 consecutive
// columns of one (batch, packed row, head); threads are ordered (row, head, column chunk) so that a warp reads whole source
// rows (the heads of a row are adjacent in the Linear / qk-norm outputs) and the row's 512-byte RoPE table is shared through
// L1 by all its heads.  The entries and their argument checks are in pf_api.cu (include/pf_b200.h pf_attn_stage_pack,
// pf_attn_varlen_pack, pf_attn_varlen_unpack).
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

// The one per-thread body of every pack kernel: 8 columns (chunk) of head h of one row for q, k and v.  The row is (stage,
// batch b, row s of the stage's sequence): text row s of text source row b * n_stages + stage for s < text_len, else video row
// row0 + s - text_len of batch b.  fr: the row's [32, 2, 2] RoPE table, or null.  packed_off: the packed element of the
// thread's first column; < 0 (backward only) when no packed row holds the source row, which then gets 0.
// kBwd = false: sources -> packed (RoPE on q, k).  kBwd = true: packed gradients -> source gradients (transposed RoPE).
template <bool kBwd, class Desc>
__device__ __forceinline__ void pack_thread(const Desc& d, int n_stages, int text_len, int stage, int b, int s, int row0,
                                            const float* fr, int h, int chunk, int64_t packed_off) {
  const bool is_text = s < text_len;
  float f[16];
  if (fr != nullptr) {
    // pairs 4 chunk .. 4 chunk + 3 of the row's [32, 2, 2] table: f[4 p + 2 c + j] multiplies x[2 p + j] into out[2 p + c]
    const float4* fr4 = reinterpret_cast<const float4*>(fr + chunk * 16);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 v = fr4[j];
      f[4 * j] = v.x; f[4 * j + 1] = v.y; f[4 * j + 2] = v.z; f[4 * j + 3] = v.w;
    }
  }

#pragma unroll
  for (int t = 0; t < 3; ++t) {
    char* src;
    bool f32;
    if (is_text) {
      const int64_t* st = d.text_strides[t];
      f32 = d.text_f32[t] != 0;
      src = static_cast<char*>(d.text[t]) +
            ((static_cast<int64_t>(b) * n_stages + stage) * st[0] + s * st[1] + h * st[2] + chunk * 8) * (f32 ? 4 : 2);
    } else {
      const int64_t* st = d.video_strides[t];
      f32 = d.video_f32[t] != 0;
      src = static_cast<char*>(d.video[t]) +
            (b * st[0] + static_cast<int64_t>(row0 + s - text_len) * st[1] + h * st[2] + chunk * 8) * (f32 ? 4 : 2);
    }
    float x[8], y[8];
    if (kBwd && packed_off < 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = 0.f;
      store8(src, f32, y);
      continue;
    }
    __nv_bfloat16* packed = static_cast<__nv_bfloat16*>(d.packed[t]) + packed_off;
    load8(kBwd ? static_cast<const void*>(packed) : src, kBwd ? false : f32, x);
    if (t < 2 && fr != nullptr) {
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

// One stage: thread (b = blockIdx.y, packed row s, head, chunk), packed [B, H, T + L, 64].
template <bool kBwd>
__global__ void __launch_bounds__(PACK_THREADS) attn_stage_pack_kernel(const pf_attn_pack_desc d) {
  const int seq = d.text_len + d.rows;
  const int i = blockIdx.x * PACK_THREADS + threadIdx.x;
  if (i >= seq * d.heads * 8) return;
  const int b = blockIdx.y;
  const int chunk = i & 7;
  const int h = (i >> 3) % d.heads;
  const int s = (i >> 3) / d.heads;
  const float* fr = d.freqs == nullptr ? nullptr : d.freqs + b * d.freqs_batch_stride + s * d.freqs_row_stride;
  const int64_t packed_off = ((static_cast<int64_t>(b) * d.heads + h) * seq + s) * PACK_HD + chunk * 8;
  pack_thread<kBwd>(d, d.n_stages, d.text_len, d.stage, b, s, d.row0, fr, h, chunk, packed_off);
}

// (stage, batch, row) of padded position p (pf_b200.h pf_attn_varlen_layout).
__device__ __forceinline__ void varlen_position(const pf_attn_varlen_layout& l, int p, int& stage, int& b, int& s) {
  stage = 0;
  while (stage + 1 < l.n_stages && p >= l.batch * l.stage_len[stage]) {
    p -= l.batch * l.stage_len[stage];
    ++stage;
  }
  b = p / l.stage_len[stage];
  s = p - b * l.stage_len[stage];
}

// Every stage of a call site: the forward runs one thread per (packed row, head, chunk), the backward one per (padded
// position, head, chunk) so that every source row is written, dropped ones with 0.  packed [1, H, total, 64].
template <bool kBwd>
__global__ void __launch_bounds__(PACK_THREADS) attn_varlen_pack_kernel(const pf_attn_varlen_pack_desc d, const int rows) {
  const pf_attn_varlen_layout& l = d.layout;
  const int i = blockIdx.x * PACK_THREADS + threadIdx.x;
  if (i >= rows * l.heads * 8) return;
  const int chunk = i & 7;
  const int h = (i >> 3) % l.heads;
  const int r = (i >> 3) / l.heads;
  const int p = kBwd ? r : l.row_map[r];
  const int packed_row = kBwd ? l.pad_map[r] : r;
  int stage, b, s;
  varlen_position(l, p, stage, b, s);
  const float* freqs = d.freqs[stage];
  const float* fr = freqs == nullptr ? nullptr : freqs + b * d.freqs_batch_stride[stage] + s * d.freqs_row_stride[stage];
  const int64_t packed_off = packed_row < 0 ? -1 : (static_cast<int64_t>(h) * l.total + packed_row) * PACK_HD + chunk * 8;
  pack_thread<kBwd>(d, l.n_stages, l.text_len, stage, b, s, l.stage_row0[stage], fr, h, chunk, packed_off);
}

// Output scatter (kBwd = false: one thread per (padded position, 8 columns), dropped rows get 0) and its gradient gather
// (kBwd = true: one thread per (packed row, 8 columns)).
template <bool kBwd>
__global__ void __launch_bounds__(PACK_THREADS) attn_varlen_unpack_kernel(const pf_attn_varlen_unpack_desc d, const int rows) {
  const pf_attn_varlen_layout& l = d.layout;
  const int width = l.heads * 8;
  const int i = blockIdx.x * PACK_THREADS + threadIdx.x;
  if (i >= rows * width) return;
  const int col = (i % width) * 8;
  const int r = i / width;
  const int p = kBwd ? l.row_map[r] : r;
  const int packed_row = kBwd ? r : l.pad_map[r];
  int stage, b, s;
  varlen_position(l, p, stage, b, s);
  char* dst;
  bool f32;
  if (s < l.text_len) {
    f32 = d.text_f32 != 0;
    dst = static_cast<char*>(d.text) +
          ((static_cast<int64_t>(b) * l.n_stages + stage) * d.text_strides[0] + s * d.text_strides[1] + col) * (f32 ? 4 : 2);
  } else {
    f32 = d.video_f32 != 0;
    dst = static_cast<char*>(d.video) +
          (b * d.video_strides[0] + static_cast<int64_t>(l.stage_row0[stage] + s - l.text_len) * d.video_strides[1] + col) *
              (f32 ? 4 : 2);
  }
  float x[8];
  if (kBwd) {
    load8(dst, f32, x);
    store8(static_cast<__nv_bfloat16*>(d.packed) + packed_row * d.ld_packed + col, false, x);
  } else {
    if (packed_row < 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j) x[j] = 0.f;
    } else {
      load8(static_cast<const __nv_bfloat16*>(d.packed) + packed_row * d.ld_packed + col, false, x);
    }
    store8(dst, f32, x);
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

static int padded_rows(const pf_attn_varlen_layout& l) {
  int64_t n = 0;
  for (int i = 0; i < l.n_stages; ++i) n += l.stage_len[i];
  return static_cast<int>(n * l.batch);
}

int attn_varlen_pack_launch(const pf_attn_varlen_pack_desc* d, bool bwd, cudaStream_t stream) {
  const int rows = bwd ? padded_rows(d->layout) : d->layout.total;
  const int64_t threads = static_cast<int64_t>(rows) * d->layout.heads * 8;
  const dim3 grid(static_cast<unsigned>((threads + PACK_THREADS - 1) / PACK_THREADS));
  if (bwd) {
    attn_varlen_pack_kernel<true><<<grid, PACK_THREADS, 0, stream>>>(*d, rows);
    return check_launch("pf_attn_varlen_pack_bwd");
  }
  attn_varlen_pack_kernel<false><<<grid, PACK_THREADS, 0, stream>>>(*d, rows);
  return check_launch("pf_attn_varlen_pack");
}

int attn_varlen_unpack_launch(const pf_attn_varlen_unpack_desc* d, bool bwd, cudaStream_t stream) {
  const int rows = bwd ? d->layout.total : padded_rows(d->layout);
  const int64_t threads = static_cast<int64_t>(rows) * d->layout.heads * 8;
  const dim3 grid(static_cast<unsigned>((threads + PACK_THREADS - 1) / PACK_THREADS));
  if (bwd) {
    attn_varlen_unpack_kernel<true><<<grid, PACK_THREADS, 0, stream>>>(*d, rows);
    return check_launch("pf_attn_varlen_unpack_bwd");
  }
  attn_varlen_unpack_kernel<false><<<grid, PACK_THREADS, 0, stream>>>(*d, rows);
  return check_launch("pf_attn_varlen_unpack");
}

}  // namespace pf
