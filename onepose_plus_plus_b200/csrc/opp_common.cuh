// opp_common.cuh — sm_90a PTX wrappers shared by every kernel of the 2D-3D matching hot path.
//
// Everything here is inline PTX for Hopper (wgmma / TMA / mbarrier / clusters). There is no
// fallback for other architectures: the translation units that include this header are
// compiled with -gencode arch=compute_90a,code=sm_90a only.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

namespace opp {

// ---------------------------------------------------------------------------------------------
// error plumbing (C-ABI functions return int status; 0 = ok)
// ---------------------------------------------------------------------------------------------
enum Status : int {
  OPP_OK = 0,
  OPP_ERR_INVALID = 1,   // bad argument (shape / alignment / null pointer)
  OPP_ERR_CUDA = 2,      // a CUDA runtime / driver call failed (see opp_last_error)
  OPP_ERR_UNSUPPORTED = 3
};

void set_last_error(const char* fmt, ...);

#define OPP_CHECK_CUDA(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::opp::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr,                 \
                            cudaGetErrorString(_e));                                      \
      return ::opp::OPP_ERR_CUDA;                                                         \
    }                                                                                     \
  } while (0)

#define OPP_REQUIRE(cond, ...)                                                            \
  do {                                                                                    \
    if (!(cond)) {                                                                        \
      ::opp::set_last_error(__VA_ARGS__);                                                 \
      return ::opp::OPP_ERR_INVALID;                                                      \
    }                                                                                     \
  } while (0)

// ---------------------------------------------------------------------------------------------
// small device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch.  Every kernel of the library is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization (launch_pdl below / launch<> in opp_gemm.cu):
// the NEXT kernel of the stream may start while this one is still running, so its launch latency
// and its prologue (barrier init, descriptor prefetch) overlap with our tail.
// Contract: each kernel calls pdl_wait() on every path before it touches global memory — it
// returns once the preceding kernel has completed and its writes are visible — and then
// pdl_trigger() so that its own successor may be scheduled.  Because every kernel waits before it
// completes, completion stays transitive along the stream.  Both are no-ops for a kernel that
// was launched without the attribute.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// OPP_PDL_TRIGGER: 0 = no explicit trigger: the successor is released when our CTAs exit, i.e. its
// launch overlaps with the end-of-grid memory flush only; 1 = trigger right after the wait (the
// successor parks early on free SMs); 2 = trigger when the main work of the CTA is done.
// 0 is the default: a grid released early by launch_dependents occupies SMs while it parks in
// griddepcontrol.wait.
#ifndef OPP_PDL_TRIGGER
#define OPP_PDL_TRIGGER 0
#endif
__device__ __forceinline__ void pdl_sync() {
  pdl_wait();
#if OPP_PDL_TRIGGER == 1
  pdl_trigger();
#endif
}
__device__ __forceinline__ void pdl_done() {
#if OPP_PDL_TRIGGER == 2
  pdl_trigger();
#endif
}

// $OPP_PDL=0 launches everything fully serialised (debugging / A-B timing)
inline int pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("OPP_PDL");
    v = e ? atoi(e) : 1;
  }
  return v;
}

// kernel<<<grid, block, smem, stream>>>(args...) with the programmatic-serialization attribute
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a mis-programmed pipeline traps (launch failure reported to the host) instead of
// hanging the GPU. ~4e9 cycles is about two seconds at H100 clocks.  No printf: any call in a
// kernel that issues wgmma makes ptxas serialise its wgmmas.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

// Lean wait for the hot MMA-issue loop: no clock reads; the watchdog counts polls instead (every
// try_wait already suspends the thread for a hardware-defined interval when the phase is pending).
__device__ __forceinline__ void mbar_wait_hot(uint64_t* bar, uint32_t parity) {
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++polls > (1u << 24)) __trap();
  }
}

// ---------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) loads; tensor maps are passed as __grid_constant__ kernel params
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* smem,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* smem,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* map, uint64_t* bar, void* smem,
                                            int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3), "r"(c4)
      : "memory");
}

// multicast variant: the box lands at the same smem offset of every CTA in `cta_mask` and performs
// complete_tx on the mbarrier at the same offset in each of them
__device__ __forceinline__ void tma_load_3d_mc(const CUtensorMap* map, uint64_t* bar, void* smem,
                                               int c0, int c1, int c2, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6}], [%2], %3;" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "h"(cta_mask), "r"(c0), "r"(c1),
      "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// thread-block clusters
// ---------------------------------------------------------------------------------------------
// arrive on the mbarrier at the same shared-memory offset in CTA `cta_rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta_rank) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta_rank)
      : "memory");
}
// the same with release semantics at cluster scope: data written to the peer's shared memory
// (st_cluster_f32x2) before the arrive is visible to a peer thread that acquires the phase
__device__ __forceinline__ void mbar_arrive_cluster_release(uint64_t* bar, uint32_t cta_rank) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta_rank)
      : "memory");
}
// two floats into CTA `cta_rank`'s shared memory, at the offset `local` has in this CTA
__device__ __forceinline__ void st_cluster_f32x2(void* local, uint32_t cta_rank, float a, float b) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "st.shared::cluster.v2.f32 [ra], {%2, %3};\n\t"
      "}\n" ::"r"(smem_u32(local)),
      "r"(cta_rank), "f"(a), "f"(b)
      : "memory");
}
// bounded wait with acquire at cluster scope (pairs with mbar_arrive_cluster_release)
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  const long long t0 = clock64();
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (ok) return;
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a): D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, fp16 operands from
// shared memory, fp32 accumulators in the registers of the 128 threads of one warpgroup
// ---------------------------------------------------------------------------------------------
// K-major operand tile in shared memory, 128-byte swizzle (what TMA SWIZZLE_128B produces for a
// box whose inner extent is 64 fp16): rows of 128 B, 8-row groups 1024 B apart.
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4 (unused: 1)
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type: 1 = SWIZZLE_128B
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// The same with 64-byte swizzle (TMA SWIZZLE_64B, inner box extent 32 fp16): rows of 64 B, 8-row
// groups 512 B apart, layout type 2.  A K step of 16 fp16 is still +32 B inside the row.
__device__ __forceinline__ uint64_t make_kmajor_sw64_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(512 >> 4) << 32;
  d |= static_cast<uint64_t>(2) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// d += A * B^T for one m64nNk16 step (both operands K-major, no transpose, unit scales).  The
// accumulator of 64 rows x N columns over the 128 threads is N/2 floats per thread: element
// 4 i + {0, 1} is row r0, columns 8 i + c0 + {0, 1}, and 4 i + {2, 3} the same columns of row r0 + 8
// (r0 = 16 * warp + lane / 4, c0 = 2 * (lane % 4)), so an n128 fragment is two n64 fragments
// concatenated.  Instantiated for the tile widths of kMmaWidths (opp_gemm.cuh).
template <int N>
__device__ __forceinline__ void wgmma_m64nNk16(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc);
#define OPP_WG_ACC8(i)                                                                              \
  "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]),    \
      "+f"(d[i + 6]), "+f"(d[i + 7])
template <>
__device__ __forceinline__ void wgmma_m64nNk16<64>(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.eq.u32 p, 0, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : OPP_WG_ACC8(0), OPP_WG_ACC8(8), OPP_WG_ACC8(16), OPP_WG_ACC8(24)
      : "l"(a_desc), "l"(b_desc)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_m64nNk16<128>(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.eq.u32 p, 0, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : OPP_WG_ACC8(0), OPP_WG_ACC8(8), OPP_WG_ACC8(16), OPP_WG_ACC8(24), OPP_WG_ACC8(32), OPP_WG_ACC8(40),
        OPP_WG_ACC8(48), OPP_WG_ACC8(56)
      : "l"(a_desc), "l"(b_desc)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_m64nNk16<208>(float (&d)[104], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.eq.u32 p, 0, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n208k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103"
      "}, %104, %105, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : OPP_WG_ACC8(0), OPP_WG_ACC8(8), OPP_WG_ACC8(16), OPP_WG_ACC8(24), OPP_WG_ACC8(32), OPP_WG_ACC8(40),
        OPP_WG_ACC8(48), OPP_WG_ACC8(56), OPP_WG_ACC8(64), OPP_WG_ACC8(72), OPP_WG_ACC8(80), OPP_WG_ACC8(88),
        OPP_WG_ACC8(96)
      : "l"(a_desc), "l"(b_desc)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_m64nNk16<256>(float (&d)[128], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.eq.u32 p, 0, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, 0, 0;\n\t"
      "}\n"
      : OPP_WG_ACC8(0), OPP_WG_ACC8(8), OPP_WG_ACC8(16), OPP_WG_ACC8(24), OPP_WG_ACC8(32), OPP_WG_ACC8(40),
        OPP_WG_ACC8(48), OPP_WG_ACC8(56), OPP_WG_ACC8(64), OPP_WG_ACC8(72), OPP_WG_ACC8(80), OPP_WG_ACC8(88),
        OPP_WG_ACC8(96), OPP_WG_ACC8(104), OPP_WG_ACC8(112), OPP_WG_ACC8(120)
      : "l"(a_desc), "l"(b_desc)
      : "memory");
}
#undef OPP_WG_ACC8
// generic-proxy shared-memory accesses ordered before later TMA (async-proxy) writes to them
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// explicit shared-space accesses (32-bit shared addresses): pointers kept in structs decay to
// generic LD/ST, which showed up as long-scoreboard stalls all over the epilogues
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "r"(addr)
               : "memory");
  return v;
}
__device__ __forceinline__ float lds32f(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts32f(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}

// register rebalancing between the warpgroups of a CTA: every warp of a warpgroup executes the same
// one; .inc waits until enough registers have been released by .dec in other warpgroups
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// named barrier among a subset of warps (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------------------------------------
// packing helpers
// ---------------------------------------------------------------------------------------------
// 16-byte global -> shared copy that bypasses the registers; src_bytes = 0 writes zeros
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
// store 8 consecutive fp16 (16 bytes) converted from fp32
__device__ __forceinline__ void store_half8(__half* dst, const float* v) {
  uint4 u;
  u.x = pack_half2(v[0], v[1]);
  u.y = pack_half2(v[2], v[3]);
  u.z = pack_half2(v[4], v[5]);
  u.w = pack_half2(v[6], v[7]);
  *reinterpret_cast<uint4*>(dst) = u;
}
__device__ __forceinline__ void load_half8(const __half* src, float* v) {
  uint4 u = *reinterpret_cast<const uint4*>(src);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __half22float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}

__device__ __forceinline__ float elu_plus_one(float x) { return x > 0.f ? x + 1.f : expf(x); }
// Epilogue variant on the SFU (ex2.approx): |rel err| <= ~(2 + |1.44 x|) ulp, i.e. < 2e-6 for the
// arguments that matter (x in (-10, 0]); one instruction pair instead of ~25.
// exp(x) as one FMUL + MUFU.EX2 (flush-to-zero): relative error ~2^-22 from ex2.approx plus
// |x| * 6e-8 from the log2(e) product, i.e. <= 1e-5 for |x| <= 100.
__device__ __forceinline__ float fast_exp(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
  return y;
}
__device__ __forceinline__ float elu_plus_one_fast(float x) { return x > 0.f ? x + 1.f : fast_exp(x); }

// ---------------------------------------------------------------------------------------------
// split-precision activations.  Every tensor that feeds a tensor-core GEMM is stored as a pair of
// fp16 planes along its channel axis: [hi(C) | lo(C)], hi = fp16(x), lo = fp16(x - hi), so that
// hi + lo carries ~22 mantissa bits.  `lo_off` is the element offset of the lo plane inside a row
// (0 = plain fp16 storage, no lo plane).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_split8(__half* row, int col, const float* v, int lo_off) {
  store_half8(row + col, v);
  if (lo_off) {
    float lo[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) lo[j] = v[j] - __half2float(__float2half_rn(v[j]));
    store_half8(row + lo_off + col, lo);
  }
}
__device__ __forceinline__ void load_split8(const __half* row, int col, float* v, int lo_off) {
  load_half8(row + col, v);
  if (lo_off) {
    float lo[8];
    load_half8(row + lo_off + col, lo);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] += lo[j];
  }
}
__device__ __forceinline__ float load_split1(const __half* row, int col, int lo_off) {
  float v = __half2float(row[col]);
  if (lo_off) v += __half2float(row[lo_off + col]);
  return v;
}
__device__ __forceinline__ void store_split1(__half* row, int col, float v, int lo_off) {
  const __half h = __float2half_rn(v);
  row[col] = h;
  if (lo_off) row[lo_off + col] = __float2half_rn(v - __half2float(h));
}

}  // namespace opp
