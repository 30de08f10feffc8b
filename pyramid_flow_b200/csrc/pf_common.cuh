// pf_common.cuh — sm_90a PTX wrappers shared by every kernel in libpf_b200.so.
//
// Everything here is a thin, hand-written wrapper over one PTX instruction:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / mma_async / commit / wait)
// and the wgmma shared-memory descriptors.  No CUTLASS/CuTe types.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pf {

// ---------------------------------------------------------------------------
// error plumbing (C-ABI: int status + pf_last_error())
// ---------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int  check_launch(const char* what);   // cudaGetLastError() -> status

#define PF_REQUIRE(cond, ...)                  \
  do {                                         \
    if (!(cond)) {                             \
      ::pf::set_error(__VA_ARGS__);            \
      return -1;                               \
    }                                          \
  } while (0)

// Driver entry point (no link-time libcuda dependency: the .so must load on a box without a GPU).
int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t rank, const void* base,
                      const uint64_t* dims, const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box,
                      CUtensorMapSwizzle swizzle,
                      const uint32_t* elem_strides = nullptr /* traversal stride per dim (strided convs); NULL = 1 */);

int num_sms();
int get_option(int key);   // pf_set_option values (include/pf_b200.h PF_OPT_*)
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device): the attribute is per device, so a process
// that drives several GPUs must set it on each (thread-safe; ~20 ns on the fast path).
int ensure_dyn_smem(const void* kernel, int bytes, const char* what);

// ---------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .b32 %%rx;\n\t"
      ".reg .pred %%px;\n\t"
      "elect.sync %%rx|%%px, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, %%px;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier -------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)   // suspend-time hint: sleep in hardware instead of polling
      : "memory");
  return ok != 0;
}
// Non-blocking probe (test_wait never suspends): lets a wait's round trip through the MIO queue overlap other work --
// issue the probe early, consume the predicate late, fall back to mbar_wait only when it was not complete yet.
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---- TMA ------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, "
      "%7}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// The box lands at the same shared-memory offset in every CTA of `cta_mask`, and each destination CTA's mbarrier at `bar`'s
// offset receives the complete_tx of its copy.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], "
      "[%2], %5;" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}

// ---- thread-block clusters ---------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// arrive on the mbarrier at `bar`'s shared-memory offset in cluster CTA `cta` (this CTA included).  Default (.release.cta)
// semantics: with .cluster scope the compiler puts a GPU-wide memory barrier in front of every arrive.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t"
      "}\n" ::"r"(smem_u32(bar)), "r"(cta)
      : "memory");
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// ---- warpgroup MMA (wgmma) ---------------------------------------------------
// One warpgroup (4 warps, 128 threads) issues D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 operands, fp32 accumulators in
// registers.  Accumulator fragment of thread (warp w, lane l), g = l / 4, t = l % 4, for every 8-column group i:
//   d[4 i + 0], d[4 i + 1] = row 16 w + g    , columns 8 i + 2 t, 8 i + 2 t + 1
//   d[4 i + 2], d[4 i + 3] = row 16 w + g + 8, same columns.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses to the accumulator registers across an asynchronous wgmma
template <int N>
__device__ __forceinline__ void wgmma_reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int REGS>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS));
}
template <int REGS>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS));
}
// named barrier over `threads` threads (ids 1.. ; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// arrive on a named barrier without waiting: counts this warp's threads towards `threads`, whose bar.sync callers it releases
__device__ __forceinline__ void named_bar_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// D[64 x 128] (+)= A[smem, K-major] * B[smem, K-major]
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
// D[64 x 128] (+)= A[smem, K-major, 64 x 32 e4m3] * B[smem, K-major, 128 x 32 e4m3]; same fragment layout as the bf16 form
__device__ __forceinline__ void wgmma_ss_n128_e4m3(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
// D[64 x 64] (+)= A[smem, K-major] * B[smem, K-major]
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
// D[64 x 64] += A[registers: 64 x 16 bf16 fragment] * B[smem, MN-major (the [k, n] tile as stored, n contiguous)]
__device__ __forceinline__ void wgmma_rs_n64_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b)
      : "memory");
}
template <int BN>
__device__ __forceinline__ void wgmma_ss(float (&d)[BN / 2], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  static_assert(BN == 128 || BN == 64, "wgmma_ss: tile widths 128 and 64 are instantiated");
  if constexpr (BN == 128) wgmma_ss_n128(d, desc_a, desc_b, accumulate);
  else wgmma_ss_n64(d, desc_a, desc_b, accumulate);
}

// ---- wgmma shared-memory descriptors -----------------------------------------
// Canonical 128B-swizzled layouts (what TMA SWIZZLE_128B writes):
//   K-major  : rows of 128 B (64 bf16 along K), 8-row atoms of 1024 B; SBO = 1024 B between 8-row groups, LBO unused.
//   MN-major : rows of 128 B (64 bf16 along M/N), 8 K-rows per 1024 B atom; SBO = 1024 B between K groups,
//              LBO = byte distance between successive 64-wide MN atoms.
// Field layout (PTX ISA "wgmma matrix descriptor"): [0,14) addr>>4, [16,30) LBO>>4, [32,46) SBO>>4, [49,52) base offset,
// [62,64) swizzle (1 = 128B).  Advancing K by 16 bf16 inside a swizzle row is +32 bytes on the start address.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ uint64_t make_smem_desc_kmajor_sw128(uint32_t saddr) {
  return make_smem_desc(saddr, 16, 1024);
}

// ---- the shared TMA -> wgmma pipeline of the GEMM and the convolution ---------
// 384 threads: warpgroup 0 = TMA producer (one elected lane), warpgroups 1, 2 = consumers, each owning 64 of the tile's 128
// rows.  Stage = A tile [128 x 64] + B tile [BN x 64], both K-major SWIZZLE_128B.  full[s]: 1 arrival + tx bytes;
// empty[s]: one arrival per consumer warp (8), made after the wgmma group that read the stage has retired.
constexpr int PIPE_THREADS = 384;
constexpr int PIPE_CONSUMER_WARPS = 8;
constexpr int PIPE_BM = 128;
constexpr int PIPE_BK = 64;
template <int BN>
struct PipeCfg {
  static constexpr int A_BYTES = PIPE_BM * PIPE_BK * 2;
  static constexpr int B_BYTES = BN * PIPE_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN >= 128) ? 4 : 6;
  static constexpr int ACC_PITCH = BN + 8;   // floats per staged accumulator row: fragment stores are bank-conflict free
  static constexpr int ACC_BYTES = PIPE_BM * ACC_PITCH * 4;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + 1024;
};

// One output tile's K loop of a consumer warpgroup: acc[64 x BN] = sum over num_kb stages.  One wgmma group stays in flight;
// a stage is handed back to the producer when the group that read it has retired.
template <int BN>
__device__ __forceinline__ void pipe_consume_tile(float (&acc)[BN / 2], uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                                  int num_kb, int wg, int& stage, uint32_t& phase) {
  using Cfg = PipeCfg<BN>;
  const int lane = threadIdx.x & 31;
  int prev = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
    const uint64_t da = make_smem_desc_kmajor_sw128(sa + wg * (64 * 128));
    const uint64_t db = make_smem_desc_kmajor_sw128(sa + Cfg::A_BYTES);
    wgmma_reg_fence(acc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < PIPE_BK / 16; ++kk) wgmma_ss<BN>(acc, da + 2 * kk, db + 2 * kk, (kb | kk) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == Cfg::STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  wgmma_reg_fence(acc);
  if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
}

// accumulator fragments of this warpgroup -> rows [64 wg, 64 wg + 64) of the fp32 staging tile (row pitch ACC_PITCH)
template <int BN>
__device__ __forceinline__ void pipe_stage_acc(const float (&acc)[BN / 2], float* acc_tile, int wg) {
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  float* r0 = acc_tile + (wg * 64 + w * 16 + (lane >> 2)) * PipeCfg<BN>::ACC_PITCH + 2 * (lane & 3);
  float* r1 = r0 + 8 * PipeCfg<BN>::ACC_PITCH;
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
    *reinterpret_cast<float2*>(r0 + 8 * i) = make_float2(acc[4 * i + 0], acc[4 * i + 1]);
    *reinterpret_cast<float2*>(r1 + 8 * i) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
  }
}

// ---- small math -----------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float rcp_approx_f(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float ex2_approx_f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_tanh_f(float x) {
  // 0.5*x*(1+tanh(u)), u = sqrt(2/pi)*(x+0.044715x^3)  ==  x*sigmoid(2u)  ==  x / (1 + 2^(-2u*log2e)).
  // 2 MUFU (ex2, rcp) + 5 FP32 ops per element, no IEEE-division slow path (that path made the GELU epilogue the
  // bottleneck of the K=1920 GEMMs); relative accuracy ~1e-6, far inside the bf16 output rounding.
  const float c0 = -2.0f * 0.7978845608028654f * 1.4426950408889634f;
  const float c1 = c0 * 0.044715f;
  const float x2 = x * x;
  const float nu = x * fmaf(x2, c1, c0);
  return x * rcp_approx_f(1.0f + ex2_approx_f(nu));
}
__device__ __forceinline__ float silu_f(float x) {
  return x * rcp_approx_f(1.0f + ex2_approx_f(-1.4426950408889634f * x));
}

}  // namespace pf
