// pf_api.cu — error plumbing, driver entry points and device queries for libpf_b200.so.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "../../include/pf_b200.h"
#include "pf_common.cuh"

namespace pf {

static thread_local char g_err[1024] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return -2;
  }
  return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
    (void)cudaGetLastError();
  });
  return fn;
}

int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t rank, const void* base,
                      const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                      CUtensorMapSwizzle swizzle, const uint32_t* elem_strides) {
  EncodeTiledFn fn = get_encode_fn();
  PF_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled is unavailable (no CUDA driver / no GPU): libpf_b200 has no CPU fallback");
  cuuint64_t gdims[5];
  cuuint64_t gstr[4];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (uint32_t i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = elem_strides ? elem_strides[i] : 1;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  CUresult r = fn(map, dtype, rank, const_cast<void*>(base), gdims, gstr, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d): rank %u dims [%llu,%llu,%llu] stride0 %llu box [%u,%u] base %p",
              static_cast<int>(r), rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 1 ? strides_bytes[0] : 0),
              box[0], rank > 1 ? box[1] : 0, base);
    return -3;
  }
  return 0;
}

int ensure_dyn_smem(const void* kernel, int bytes, const char* what) {
  struct Entry { const void* k; unsigned long long devmask; };
  static std::mutex mu;
  static Entry table[128];
  static int n_entries = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("%s: no CUDA device", what);
    return -2;
  }
  const unsigned long long bit = 1ull << (dev & 63);
  std::lock_guard<std::mutex> lock(mu);
  Entry* e = nullptr;
  for (int i = 0; i < n_entries; ++i)
    if (table[i].k == kernel) { e = &table[i]; break; }
  if (e != nullptr && (e->devmask & bit)) return 0;
  cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (err != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("cudaFuncSetAttribute(%s, dynamic smem %d): %s", what, bytes, cudaGetErrorString(err));
    return -2;
  }
  if (e == nullptr && n_entries < 128) { e = &table[n_entries++]; e->k = kernel; e->devmask = 0; }
  if (e != nullptr) e->devmask |= bit;
  return 0;
}

// Library options (pf_set_option): new data paths stay opt-in until a hardware run has validated them; the defaults below are
// the validated choices.
static std::atomic<int> g_options[PF_OPT_COUNT] = {};
static std::once_flag g_options_once;
static void options_init() {
  g_options[PF_OPT_GEMM_STAGED_RESID].store(PF_OPT_DEFAULT_GEMM_STAGED_RESID);
  g_options[PF_OPT_GEMM_WAVE_TILING].store(PF_OPT_DEFAULT_GEMM_WAVE_TILING);
  g_options[PF_OPT_ATTN_PAIR_KERNEL].store(PF_OPT_DEFAULT_ATTN_PAIR_KERNEL);
  g_options[PF_OPT_ATTN_TILE_PHASE].store(PF_OPT_DEFAULT_ATTN_TILE_PHASE);
  g_options[PF_OPT_ATTN_TRIPLE_KERNEL].store(PF_OPT_DEFAULT_ATTN_TRIPLE_KERNEL);
}
int get_option(int key) {
  std::call_once(g_options_once, options_init);
  return (key >= 0 && key < PF_OPT_COUNT) ? g_options[key].load(std::memory_order_relaxed) : 0;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return 0;
    n = prop.multiProcessorCount;
  }
  return n;
}

int warmup_gemm();
int warmup_conv();
int warmup_conv_bwd();
int warmup_attn();
int warmup_text();
int attn_stage_pack_launch(const pf_attn_pack_desc* d, bool bwd, cudaStream_t stream);   // pf_attn_pack.cu
int attn_varlen_pack_launch(const pf_attn_varlen_pack_desc* d, bool bwd, cudaStream_t stream);
int attn_varlen_unpack_launch(const pf_attn_varlen_unpack_desc* d, bool bwd, cudaStream_t stream);

static int check_pack_source(const char* what, const char* name, int t, const void* p, const int64_t* strides, int32_t is_f32) {
  PF_REQUIRE(p != nullptr, "%s: %s[%d] is null", what, name, t);
  PF_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15) == 0, "%s: %s[%d] is not 16-byte aligned", what, name, t);
  PF_REQUIRE(is_f32 == 0 || is_f32 == 1, "%s: %s_f32[%d] = %d (0 = bf16, 1 = fp32)", what, name, t, is_f32);
  for (int i = 0; i < 3; ++i)
    PF_REQUIRE(strides[i] > 0 && strides[i] % 8 == 0, "%s: %s[%d] stride %d = %lld, needs a positive multiple of 8 elements",
               what, name, t, i, static_cast<long long>(strides[i]));
  return 0;
}

// Everything the pack kernels address, checked before any launch.
static int check_pack_desc(const pf_attn_pack_desc* d, const char* what) {
  PF_REQUIRE(d != nullptr, "%s: null descriptor", what);
  PF_REQUIRE(d->head_dim == 64, "%s: head_dim %d unsupported (64 only)", what, d->head_dim);
  PF_REQUIRE(d->batch > 0 && d->batch <= 65535 && d->heads > 0 && d->rows > 0 && d->text_len >= 0,
             "%s: bad shape (batch %d, heads %d, rows %d, text_len %d)", what, d->batch, d->heads, d->rows, d->text_len);
  PF_REQUIRE(d->row0 >= 0 && static_cast<int64_t>(d->row0) + d->rows <= d->src_rows,
             "%s: stage rows [%d, %lld) outside the source's %d rows", what, d->row0,
             static_cast<long long>(d->row0) + d->rows, d->src_rows);
  PF_REQUIRE((static_cast<int64_t>(d->text_len) + d->rows) * d->heads * 8 < (int64_t(1) << 31),
             "%s: stage too large (%d rows x %d heads)", what, d->text_len + d->rows, d->heads);
  for (int t = 0; t < 3; ++t) {
    PF_REQUIRE(d->packed[t] != nullptr && (reinterpret_cast<uintptr_t>(d->packed[t]) & 15) == 0,
               "%s: packed[%d] null or not 16-byte aligned", what, t);
    if (int rc = check_pack_source(what, "video", t, d->video[t], d->video_strides[t], d->video_f32[t])) return rc;
  }
  if (d->text_len > 0) {
    PF_REQUIRE(d->n_stages > 0 && d->stage >= 0 && d->stage < d->n_stages, "%s: stage %d of %d", what, d->stage, d->n_stages);
    for (int t = 0; t < 3; ++t)
      if (int rc = check_pack_source(what, "text", t, d->text[t], d->text_strides[t], d->text_f32[t])) return rc;
  }
  if (d->freqs != nullptr)
    PF_REQUIRE((reinterpret_cast<uintptr_t>(d->freqs) & 15) == 0 && d->freqs_batch_stride > 0 && d->freqs_batch_stride % 4 == 0 &&
                   d->freqs_row_stride >= 128 && d->freqs_row_stride % 4 == 0,
               "%s: freqs must be 16-byte aligned with strides multiples of 4 and a row stride >= 128 (batch %lld, row %lld)",
               what, static_cast<long long>(d->freqs_batch_stride), static_cast<long long>(d->freqs_row_stride));
  return 0;
}

// The stage layout shared by the varlen pack and unpack entries (the maps' contents are the caller's, see pf_b200.h).
static int check_varlen_layout(const pf_attn_varlen_layout& l, const char* what) {
  PF_REQUIRE(l.head_dim == 64, "%s: head_dim %d unsupported (64 only)", what, l.head_dim);
  PF_REQUIRE(l.batch > 0 && l.heads > 0 && l.text_len >= 0 && l.src_rows > 0 && l.total > 0,
             "%s: bad shape (batch %d, heads %d, text_len %d, src_rows %d, total %d)", what, l.batch, l.heads, l.text_len,
             l.src_rows, l.total);
  PF_REQUIRE(l.n_stages >= 1 && l.n_stages <= PF_ATTN_VARLEN_MAX_STAGES, "%s: n_stages %d not in [1, %d]", what, l.n_stages,
             PF_ATTN_VARLEN_MAX_STAGES);
  int64_t padded = 0;
  for (int i = 0; i < l.n_stages; ++i) {
    PF_REQUIRE(l.stage_len[i] > l.text_len && l.stage_row0[i] >= 0 &&
                   static_cast<int64_t>(l.stage_row0[i]) + l.stage_len[i] - l.text_len <= l.src_rows,
               "%s: stage %d (%d rows from video row %d, text_len %d) outside the source's %d rows", what, i, l.stage_len[i],
               l.stage_row0[i], l.text_len, l.src_rows);
    padded += static_cast<int64_t>(l.stage_len[i]) * l.batch;
  }
  PF_REQUIRE(l.total <= padded, "%s: total %d exceeds the %lld padded rows", what, l.total, static_cast<long long>(padded));
  PF_REQUIRE(padded * l.heads * 8 < (int64_t(1) << 31), "%s: too large (%lld padded rows x %d heads)", what,
             static_cast<long long>(padded), l.heads);
  PF_REQUIRE(l.row_map != nullptr && l.pad_map != nullptr && (reinterpret_cast<uintptr_t>(l.row_map) & 3) == 0 &&
                 (reinterpret_cast<uintptr_t>(l.pad_map) & 3) == 0,
             "%s: row_map / pad_map null or not 4-byte aligned", what);
  return 0;
}

static int check_varlen_pack_desc(const pf_attn_varlen_pack_desc* d, const char* what) {
  PF_REQUIRE(d != nullptr, "%s: null descriptor", what);
  const pf_attn_varlen_layout& l = d->layout;
  if (int rc = check_varlen_layout(l, what)) return rc;
  for (int t = 0; t < 3; ++t) {
    PF_REQUIRE(d->packed[t] != nullptr && (reinterpret_cast<uintptr_t>(d->packed[t]) & 15) == 0,
               "%s: packed[%d] null or not 16-byte aligned", what, t);
    if (int rc = check_pack_source(what, "video", t, d->video[t], d->video_strides[t], d->video_f32[t])) return rc;
    if (l.text_len > 0)
      if (int rc = check_pack_source(what, "text", t, d->text[t], d->text_strides[t], d->text_f32[t])) return rc;
  }
  for (int i = 0; i < l.n_stages; ++i)
    if (d->freqs[i] != nullptr)
      PF_REQUIRE((reinterpret_cast<uintptr_t>(d->freqs[i]) & 15) == 0 && d->freqs_batch_stride[i] > 0 &&
                     d->freqs_batch_stride[i] % 4 == 0 && d->freqs_row_stride[i] >= 128 && d->freqs_row_stride[i] % 4 == 0,
                 "%s: freqs[%d] must be 16-byte aligned with strides multiples of 4 and a row stride >= 128 (batch %lld, row %lld)",
                 what, i, static_cast<long long>(d->freqs_batch_stride[i]), static_cast<long long>(d->freqs_row_stride[i]));
  return 0;
}

static int check_unpack_rows(const char* what, const char* name, const void* p, const int64_t* strides, int32_t is_f32,
                             int32_t heads) {
  PF_REQUIRE(p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0, "%s: %s null or not 16-byte aligned", what, name);
  PF_REQUIRE(is_f32 == 0 || is_f32 == 1, "%s: %s_f32 = %d (0 = bf16, 1 = fp32)", what, name, is_f32);
  PF_REQUIRE(strides[0] > 0 && strides[0] % 8 == 0 && strides[1] % 8 == 0 && strides[1] >= static_cast<int64_t>(heads) * 64,
             "%s: %s strides (batch %lld, row %lld) need positive multiples of 8 elements and a row stride >= %d", what, name,
             static_cast<long long>(strides[0]), static_cast<long long>(strides[1]), heads * 64);
  return 0;
}

static int check_varlen_unpack_desc(const pf_attn_varlen_unpack_desc* d, const char* what) {
  PF_REQUIRE(d != nullptr, "%s: null descriptor", what);
  const pf_attn_varlen_layout& l = d->layout;
  if (int rc = check_varlen_layout(l, what)) return rc;
  PF_REQUIRE(d->packed != nullptr && (reinterpret_cast<uintptr_t>(d->packed) & 15) == 0 && d->ld_packed % 8 == 0 &&
                 d->ld_packed >= static_cast<int64_t>(l.heads) * 64,
             "%s: packed null, not 16-byte aligned, or ld_packed %lld not a multiple of 8 >= %d", what,
             static_cast<long long>(d->ld_packed), l.heads * 64);
  if (int rc = check_unpack_rows(what, "video", d->video, d->video_strides, d->video_f32, l.heads)) return rc;
  if (l.text_len > 0)
    if (int rc = check_unpack_rows(what, "text", d->text, d->text_strides, d->text_f32, l.heads)) return rc;
  return 0;
}

}  // namespace pf

extern "C" {

// ---- pf_ctx: a recorded launch sequence (one DiT step, one VAE chunk ...) owned by the library ---------------------------
struct pf_ctx {
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  cudaStream_t rec_stream = nullptr;
  bool recording = false;
  size_t nodes = 0;
};

int pf_ctx_create(pf_ctx** out) {
  if (out == nullptr) {
    pf::set_error("pf_ctx_create: null");
    return -1;
  }
  *out = new pf_ctx();
  return 0;
}

static void ctx_drop(pf_ctx* c) {
  if (c->exec) cudaGraphExecDestroy(c->exec);
  if (c->graph) cudaGraphDestroy(c->graph);
  c->exec = nullptr;
  c->graph = nullptr;
  c->nodes = 0;
}

int pf_ctx_destroy(pf_ctx* c) {
  if (c == nullptr) return 0;
  if (c->recording) {
    cudaGraph_t g = nullptr;
    cudaStreamEndCapture(c->rec_stream, &g);
    if (g) cudaGraphDestroy(g);
  }
  ctx_drop(c);
  (void)cudaGetLastError();
  delete c;
  return 0;
}

int pf_ctx_record_begin(pf_ctx* c, void* stream) {
  using namespace pf;
  PF_REQUIRE(c != nullptr && !c->recording, "pf_ctx_record_begin: null context or already recording");
  int rc = pf_warmup();          // nothing may initialise host-side while the stream is capturing
  if (rc) return rc;
  ctx_drop(c);
  c->rec_stream = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaStreamBeginCapture(c->rec_stream, cudaStreamCaptureModeThreadLocal);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("pf_ctx_record_begin: cudaStreamBeginCapture: %s", cudaGetErrorString(e));
    return -2;
  }
  c->recording = true;
  return 0;
}

int pf_ctx_record_end(pf_ctx* c) {
  using namespace pf;
  PF_REQUIRE(c != nullptr && c->recording, "pf_ctx_record_end: not recording");
  c->recording = false;
  cudaError_t e = cudaStreamEndCapture(c->rec_stream, &c->graph);
  if (e == cudaSuccess) e = cudaGraphGetNodes(c->graph, nullptr, &c->nodes);
  if (e == cudaSuccess) e = cudaGraphInstantiate(&c->exec, c->graph, 0);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    ctx_drop(c);
    set_error("pf_ctx_record_end: %s", cudaGetErrorString(e));
    return -2;
  }
  return static_cast<int>(c->nodes);
}

int pf_ctx_replay(pf_ctx* c, void* stream) {
  using namespace pf;
  PF_REQUIRE(c != nullptr && c->exec != nullptr, "pf_ctx_replay: nothing recorded");
  cudaError_t e = cudaGraphLaunch(c->exec, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("pf_ctx_replay: cudaGraphLaunch: %s", cudaGetErrorString(e));
    return -2;
  }
  g_launches.fetch_add(static_cast<int64_t>(c->nodes), std::memory_order_relaxed);
  return 0;
}

int pf_dit_step_flux(pf_ctx* c, void* stream) { return pf_ctx_replay(c, stream); }
int pf_dit_step_mmdit(pf_ctx* c, void* stream) { return pf_ctx_replay(c, stream); }
int pf_vae_decode_chunk(pf_ctx* c, void* stream) { return pf_ctx_replay(c, stream); }

int pf_attn_stage_pack(const pf_attn_pack_desc* d, void* stream) {
  if (int rc = pf::check_pack_desc(d, "pf_attn_stage_pack")) return rc;
  return pf::attn_stage_pack_launch(d, false, static_cast<cudaStream_t>(stream));
}

int pf_attn_stage_pack_bwd(const pf_attn_pack_desc* d, void* stream) {
  if (int rc = pf::check_pack_desc(d, "pf_attn_stage_pack_bwd")) return rc;
  return pf::attn_stage_pack_launch(d, true, static_cast<cudaStream_t>(stream));
}

int pf_attn_varlen_pack(const pf_attn_varlen_pack_desc* d, void* stream) {
  if (int rc = pf::check_varlen_pack_desc(d, "pf_attn_varlen_pack")) return rc;
  return pf::attn_varlen_pack_launch(d, false, static_cast<cudaStream_t>(stream));
}

int pf_attn_varlen_pack_bwd(const pf_attn_varlen_pack_desc* d, void* stream) {
  if (int rc = pf::check_varlen_pack_desc(d, "pf_attn_varlen_pack_bwd")) return rc;
  return pf::attn_varlen_pack_launch(d, true, static_cast<cudaStream_t>(stream));
}

int pf_attn_varlen_unpack(const pf_attn_varlen_unpack_desc* d, void* stream) {
  if (int rc = pf::check_varlen_unpack_desc(d, "pf_attn_varlen_unpack")) return rc;
  return pf::attn_varlen_unpack_launch(d, false, static_cast<cudaStream_t>(stream));
}

int pf_attn_varlen_unpack_bwd(const pf_attn_varlen_unpack_desc* d, void* stream) {
  if (int rc = pf::check_varlen_unpack_desc(d, "pf_attn_varlen_unpack_bwd")) return rc;
  return pf::attn_varlen_unpack_launch(d, true, static_cast<cudaStream_t>(stream));
}

int pf_set_option(int key, int value) {
  std::call_once(pf::g_options_once, pf::options_init);
  if (key < 0 || key >= PF_OPT_COUNT) {
    pf::set_error("pf_set_option: unknown key %d", key);
    return -1;
  }
  pf::g_options[key].store(value);
  return 0;
}
int pf_get_option(int key) { return pf::get_option(key); }

int pf_warmup(void) {
  int rc = pf::warmup_gemm();
  if (!rc) rc = pf::warmup_conv();
  if (!rc) rc = pf::warmup_conv_bwd();
  if (!rc) rc = pf::warmup_attn();
  if (!rc) rc = pf::warmup_text();
  return rc;
}

const char* pf_last_error(void) { return pf::g_err; }
int pf_version(void) { return 202; }
int64_t pf_launch_count(void) { return pf::g_launches.load(); }

int pf_device_check(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    pf::set_error("no CUDA device: %s", cudaGetErrorString(e));
    return -1;
  }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    pf::set_error("cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    return -1;
  }
  if (prop.major != 9) {
    pf::set_error("libpf_b200 is built for sm_90a only; device is sm_%d%d", prop.major, prop.minor);
    return -1;
  }
  if (pf::get_encode_fn() == nullptr) {
    pf::set_error("driver does not expose cuTensorMapEncodeTiled");
    return -1;
  }
  return 0;
}

}  // extern "C"
