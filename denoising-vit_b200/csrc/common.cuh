// Common device/host helpers for the dvt_b200 kernels (sm_90a: H100).
//
// Thin inline-PTX wrappers for mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma) and the fence between
// the generic and async proxies.  Every blocking wait in this file is
// bounded by a clock watchdog: a kernel that would dead-lock records a code in g_dvt_dev_error and traps
// instead of hanging the GPU.
#pragma once

#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>

#ifndef DVT_WATCHDOG_CYCLES
#define DVT_WATCHDOG_CYCLES 4000000000ll  // ~2 s at 1.9 GHz
#endif

namespace dvt {

// ------------------------------------------------------------------------------------------------
// host-side error plumbing (api.cu owns the storage)
// ------------------------------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define DVT_CUDA_OK(expr)                                                        \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) return ::dvt::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)

#define DVT_REQUIRE(cond, ...)                    \
  do {                                            \
    if (!(cond)) {                                \
      ::dvt::set_last_error(__VA_ARGS__);         \
      return DVT_ERR_INVALID;                     \
    }                                             \
  } while (0)

enum { DVT_OK = 0, DVT_ERR_INVALID = 1, DVT_ERR_CUDA = 2, DVT_ERR_DEVICE = 3 };

// device-side error word: 0 = fine; otherwise (code << 16 | detail)
// (defined here: the library is built as ONE translation unit, see dvt_b200_all.cu)
__device__ unsigned int g_dvt_dev_error = 0;

// ------------------------------------------------------------------------------------------------
// small device utilities
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() {
  uint32_t l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void dev_fail(unsigned code, unsigned detail) {
  atomicCAS(&g_dvt_dev_error, 0u, (code << 16) | (detail & 0xffffu));
  __threadfence_system();
  __trap();
}

// ------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// (A suspend-time hint on try_wait -- `mbarrier.try_wait ..., hint_ns` -- was measured in round 2: no effect on the attention
// kernel, 0.365 -> 0.368 ms, and the fit's step chain got slower, so the plain form stays.)
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

// Bounded wait: traps (instead of hanging) when the phase never completes.
// Wait of a role that is not latency critical (a TMA producer waiting for a free slot): backs off with nanosleep so that
// its spin loop does not take issue slots from the math warps on the same scheduler.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity, unsigned tag = 0) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(64);
    if (clock64() - t0 > DVT_WATCHDOG_CYCLES) dev_fail(0xDEADu, tag);
  }
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, unsigned tag = 0) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > DVT_WATCHDOG_CYCLES) dev_fail(0xDEADu, tag);
  }
}

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ------------------------------------------------------------------------------------------------
// programmatic dependent launch (PDL): a kernel launched with launch_k(pdl = true, ...) may start -- block scheduling,
// barrier set-up -- while the previous kernel of its stream is still running; pdl_wait() blocks until that kernel
// has completed and its writes are visible, pdl_trigger() lets the NEXT kernel of the stream start its own prologue.
// Both are no-ops in a kernel that was launched without the attribute.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// prio_drop > 0: the kernel runs that many levels BELOW the highest stream priority whatever its stream's priority is
// (kernels off the critical path that would otherwise take the SMs the next critical kernel is waiting for).
struct LaunchOpt {
  bool pdl = false;
  int prio_drop = 0;
};
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kx(LaunchOpt o, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                             Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (o.pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (o.prio_drop > 0) {
    static int lo = 0, hi = 0;
    static const cudaError_t range_rc = cudaDeviceGetStreamPriorityRange(&lo, &hi);  // (numerically lower = higher priority)
    if (range_rc != cudaSuccess) return range_rc;
    attr[na].id = cudaLaunchAttributePriority;
    attr[na].val.priority = hi + o.prio_drop < lo ? hi + o.prio_drop : lo;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(bool pdl, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                            Args&&... args) {
  return launch_kx(LaunchOpt{pdl, 0}, kern, grid, block, smem, st, static_cast<Args&&>(args)...);
}

// ------------------------------------------------------------------------------------------------
// proxy fence
// ------------------------------------------------------------------------------------------------
// generic-proxy smem writes -> visible to the async proxy (TMA store / wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ------------------------------------------------------------------------------------------------
// TMA (tiled mode).  Coordinates are innermost-first.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// 1-D bulk copy global -> shared (no tensor map): size and both addresses multiples of 16 bytes
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): D[64 x N] (+)= A[64 x K] * B[K x N], fp32 accumulators in registers.
// Issued by all 128 threads of a warpgroup (4 consecutive warps, the first one's index a multiple of 4).
// Accumulator layout (thread t = 32 w + l of the warpgroup): d[4 j + 2 i + c] = D[16 w + l / 4 + 8 i][8 j + 2 (l % 4) + c].
// ------------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle (the layout TMA writes with CU_TENSOR_MAP_SWIZZLE_128B).
//   K-major operand: rows of 128 B, 8-row groups `sbo` = 1024 B apart; K advances 32 B (+2 in the descriptor) per MMA.
//   MN-major operand (bf16 only): [MN / 64 atoms, `lbo` bytes apart][K rows of 128 B, 8-row groups `sbo` apart].
__device__ __forceinline__ uint64_t make_wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= 1ull << 62;  // layout type: 128B swizzle
  return d;
}
// The same descriptor for the 32-byte swizzle (CU_TENSOR_MAP_SWIZZLE_32B: rows of 32 B = 16 bf16, 8-row atoms of 256 B).
//   K-major operand: one k16 step per 32-byte row; 8-row groups `sbo` = 256 B apart.
//   MN-major operand: [MN / 16 atoms, `lbo` bytes apart][K rows of 32 B, 8-row groups `sbo` = 256 B apart].
__device__ __forceinline__ uint64_t make_wgmma_desc_sw32(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= 3ull << 62;  // layout type: 32B swizzle
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accumulator reads / writes across an in-flight wgmma.
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D (+)= A . B, both from shared memory; TA / TB: 1 = MN-major operand (bf16 only).  Always accumulates: zero D first.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_128_bf16(float (&d)[64], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(1), "n"(TA), "n"(TB));
}

__device__ __forceinline__ void wgmma_128_tf32(float (&d)[64], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(1));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_64_bf16(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(1), "n"(TA), "n"(TB));
}

template <int TB>
__device__ __forceinline__ void wgmma_64_bf16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1), "n"(TB));
}

// m64n32k16 (half a 64-query tile of the head_dim-80 attention backward): 16 accumulators per thread.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_32_bf16(float (&d)[16], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(1), "n"(TA), "n"(TB));
}

// m64n16k16 forms (the 16-column tail of head_dim 80): D[64 x 16], 8 accumulators per thread.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_16_bf16(float (&d)[8], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(1), "n"(TA), "n"(TB));
}

template <int TB>
__device__ __forceinline__ void wgmma_16_bf16_rs(float (&d)[8], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, %14;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(1), "n"(TB));
}

// named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ------------------------------------------------------------------------------------------------
// math helpers
// ------------------------------------------------------------------------------------------------
// fp32 pairs: two independent fp32 operations, each rounded exactly like its scalar form (the GELU epilogue and the softmax
// are written on pairs).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// erf with ONE transcendental: erfc(t) = 2^q(t) for t = |x|, q a degree-6 polynomial without constant term fitted to
// log2(erfc(t)) on [0, 4.2] (weighted so that the absolute error of erf is minimised: max |err| 3.3e-7 in fp32, evaluated
// against scipy.special.erf on 2e5 points); erf(x) = sign(x) (1 - 2^q).  t is clamped to 6 (erfc(6) = 2e-17 rounds 1 - e
// to 1; the polynomial turns upward far outside its fitting range).  Round 1 used Abramowitz-Stegun 7.1.26 (a reciprocal
// AND an exponential per element): in the fc1 + GELU epilogue the MUFU pipe -- 2 ops x 32 768 elements per tile -- cost
// 2/3 of the tile's MMA time.
__device__ __forceinline__ float fast_erf(float x) {
  const float t = fminf(fabsf(x), 6.0f);
  float q = 1.580459628734477e-4f;
  q = fmaf(q, t, -3.742739173536956e-3f);
  q = fmaf(q, t, 3.1032528216293022e-2f);
  q = fmaf(q, t, -1.498016394645605e-1f);
  q = fmaf(q, t, -9.181337298819333e-1f);
  q = fmaf(q, t, -1.6279281218285298f);
  q *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(q));
  return copysignf(1.0f - e, x);
}
// GELU(x) = x Phi(x) = max(x, 0) - 0.5 |x| erfc(|x| / sqrt 2): with erfc = 2^q as in fast_erf (same polynomial, written in
// a = |x| with the -1 of the factor 0.5 folded into the exponent) this is 11 instructions per element instead of 18 -- the
// fc1 epilogue is issue bound (ncu: issue 50 %, tensor 51 %).  Max abs error vs the exact erf GELU 5.2e-7.
__device__ __forceinline__ float gelu_erf(float x) {
  const float a = fminf(fabsf(x), 8.485281374f);
  float q = 1.9755745359180961e-05f;
  q = fmaf(q, a, -6.6162906245512902e-04f);
  q = fmaf(q, a, 7.7581320540732555e-03f);
  q = fmaf(q, a, -5.2962877549126521e-02f);
  q = fmaf(q, a, -4.5906686494096666e-01f);
  q = fmaf(q, a, -1.1511190142292334f);
  q = fmaf(q, a, -1.0f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(q));
  return fmaf(-a, e, fmaxf(x, 0.0f));
}

// Two GELUs in packed fp32 pairs: the polynomial is evaluated in n = -min(|x|, 8.485) (one FMNMX with source modifiers; the
// odd coefficients change sign, every intermediate is the exact negation or copy of the scalar form's, so the result is
// bit-identical to gelu_erf).
__device__ __forceinline__ float2 gelu_erf2(float2 x) {
  const float2 n = make_float2(fmaxf(-fabsf(x.x), -8.485281374f), fmaxf(-fabsf(x.y), -8.485281374f));
  float2 q = make_float2(1.9755745359180961e-05f, 1.9755745359180961e-05f);
  q = ffma2(q, n, make_float2(6.6162906245512902e-04f, 6.6162906245512902e-04f));
  q = ffma2(q, n, make_float2(7.7581320540732555e-03f, 7.7581320540732555e-03f));
  q = ffma2(q, n, make_float2(5.2962877549126521e-02f, 5.2962877549126521e-02f));
  q = ffma2(q, n, make_float2(-4.5906686494096666e-01f, -4.5906686494096666e-01f));
  q = ffma2(q, n, make_float2(1.1511190142292334f, 1.1511190142292334f));
  q = ffma2(q, n, make_float2(-1.0f, -1.0f));
  float2 e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(q.x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(q.y));
  return ffma2(n, e, make_float2(fmaxf(x.x, 0.0f), fmaxf(x.y, 0.0f)));
}

// d/dx gelu_erf(x) = Phi(x) + x phi(x)
__device__ __forceinline__ float gelu_grad(float x) {
  return fmaf(x * 0.3989422804014327f, __expf(-0.5f * x * x), 0.5f * (1.0f + fast_erf(x * 0.70710678118654752f)));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------------
// host: TMA descriptor creation (driver entry point resolved at run time; no link against libcuda)
// ------------------------------------------------------------------------------------------------
enum TmapDtype { TMAP_BF16 = 0, TMAP_F32 = 1 };
// 2-D row-major tensor [rows, cols] with `row_pitch_bytes`; box = [box_rows, box_cols]; 128B swizzle.
int make_tmap_2d(CUtensorMap* out, const void* base, TmapDtype dt, uint64_t rows, uint64_t cols,
                 uint64_t row_pitch_bytes, uint32_t box_rows, uint32_t box_cols);
// 3-D tensor [d2, d1, d0(contiguous)] with byte strides for d1 and d2; box = [1, box1, box0].  swizzle_bytes: 128
// (default) or 32 (boxes of 32-byte rows: the 16-column tail slab of the head_dim-80 attention tiles).
int make_tmap_3d(CUtensorMap* out, const void* base, TmapDtype dt, uint64_t d0, uint64_t d1, uint64_t d2,
                 uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t box0, uint32_t box1, uint32_t box2 = 1,
                 int swizzle_bytes = 128);

int num_sms();

// host-side tally of kernels launched by this library (graph replays add the node count of the graph)
void count_launch(long long n = 1);
// Set by vit_forward around its block loop: LayerNorm / attention launches then use programmatic dependent launch (each
// process drives one GPU from one thread, see INTEGRATION.md).
extern bool g_vit_pdl;
long long launch_count();

}  // namespace dvt
