// wgmma / TMA / mbarrier PTX wrappers and tile constants shared by the tensor-core kernels (sm_90a).
#pragma once
#include <cuda.h>
#include "common.cuh"
#include <cuda_fp16.h>
#include "wgmma.cuh"

namespace dasr {

constexpr int TILE_H = 16, TILE_W = 8;
constexpr int HALO_H = TILE_H + 2, HALO_W = TILE_W + 2;
constexpr int CHUNK = 32;                      // channels per K chunk (64 B rows, SWIZZLE_64B)
constexpr int ROW_B = CHUNK * 2;               // 64
constexpr int A_HALO_BYTES = HALO_H * HALO_W * ROW_B;   // 11520
constexpr int A_TAP_BYTES = TILE_H * TILE_W * ROW_B;    // 8192 (a_mode 1: one aligned tile per tap)
constexpr int MAX_STAGES = 8;
constexpr int SMEM_LIMIT = 226 * 1024;  // 227 KB opt-in max minus the kernel's 1 KB static allocation

// ---------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- warpgroup MMA (wgmma) synchronisation ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across a wgmma fence or wait
template <int R>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// sm_90 shared-memory matrix descriptor: [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) layout
// (1 = SWIZZLE_128B, 2 = SWIZZLE_64B).  K-major swizzled operands ignore LBO (1); MN-major ones use it as the stride
// between swizzle-width groups of the M / N index.  The swizzle is a function of the shared-memory address bits, as it is
// for the TMA writes, so a start address shifted by whole 64 B / 128 B rows (a conv tap) reads the tile TMA wrote.
constexpr uint64_t DESC_SW128 = (uint64_t)1 << 62;
constexpr uint64_t DESC_SW64 = (uint64_t)2 << 62;
__device__ __forceinline__ uint64_t desc_hi(uint32_t lbo, uint32_t sbo, uint64_t layout) {
  return ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo >> 4) & 0x3FFF) << 32) | layout;
}
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint64_t hi) { return hi | (uint64_t)((smem_addr >> 4) & 0x3FFF); }

// ---- thread-block clusters ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at the same shared-memory offset in cluster CTA `rank`
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// TMA load written to the same shared-memory offset of every CTA in `mask`; each destination's barrier at `bar`'s offset
// receives the bytes it got
__device__ __forceinline__ void tma_load_4d_mc(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                               int c3, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "h"(mask)
      : "memory");
}
// programmatic dependent launch: wait for the prerequisite grid's memory / let the dependent grid start its prologue
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// TMA store / bulk-group helpers (epilogue)
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Warp-wide: wait until every CTA k < g of a producer launch has finished all of its tiles with raster index <= tmax
// (CTA k owns tiles k, k+g, k+2g, ...).  Progress is monotone, so a satisfied bound never has to be re-checked.
__device__ __forceinline__ void wait_producer(const int* prog, int g, long tmax, int lane) {
  if (prog == nullptr) return;
  for (int base = 0; base < g; base += 32) {
    const int k = base + lane;
    const int need = (k < g && tmax >= k) ? (int)((tmax - k) / g) + 1 : 0;
    while (true) {
      const int v = (k < g) ? ld_acquire_gpu(prog + k) : 0x7fffffff;
      if (__all_sync(0xffffffffu, v >= need)) break;
      __nanosleep(100);
    }
  }
  asm volatile("fence.proxy.async;" ::: "memory");   // generic-proxy acquire -> subsequent TMA (async proxy) reads
}

// explicit shared-space 128-bit accesses with 32-bit addresses (generic pointers cost 64-bit address math + LD.E)
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float4 lds128f(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}

constexpr int EPI_BLK64_BYTES = 128 * 128;   // 64-channel block of a staged tile: 128 pixels x 128 B, SWIZZLE_128B
constexpr int EPI_BLK32_BYTES = 128 * 64;    // 32-channel tail block:            128 pixels x  64 B, SWIZZLE_64B

__device__ __forceinline__ void fma_bf16x8(float* v, const uint4& u, float s) {
  const __nv_bfloat162* b2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int j = 0; j < 4; j++) {
    float2 f = __bfloat1622float2(b2[j]);
    v[2 * j] = fmaf(s, f.x, v[2 * j]);
    v[2 * j + 1] = fmaf(s, f.y, v[2 * j + 1]);
  }
}

// v[0..8) += s * (8 packed 16-bit values of u), bf16 or IEEE half
__device__ __forceinline__ void fma_h16x8(float* v, const uint4& u, float s, int f16) {
  if (f16) {
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      float2 f = __half22float2(h2[j]);
      v[2 * j] = fmaf(s, f.x, v[2 * j]);
      v[2 * j + 1] = fmaf(s, f.y, v[2 * j + 1]);
    }
  } else {
    fma_bf16x8(v, u, s);
  }
}
// 16 floats -> 16 packed 16-bit values (round to nearest even)
__device__ __forceinline__ void pack_h16x16(const float* v, uint4* o, int f16) {
  if (f16) {
    __half2* oh = reinterpret_cast<__half2*>(o);
#pragma unroll
    for (int j = 0; j < 8; j++) oh[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
  } else {
    __nv_bfloat162* ob = reinterpret_cast<__nv_bfloat162*>(o);
#pragma unroll
    for (int j = 0; j < 8; j++) ob[j] = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

}  // namespace dasr
