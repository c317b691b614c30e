// sm_90a building blocks: mbarrier, TMA (cp.async.bulk.tensor) and warpgroup MMA (wgmma) wrappers as
// inline PTX, the shared-memory matrix descriptors the tensor-core kernels share, and the accumulator
// transposition that hands a 128-row wgmma accumulator to row-per-thread epilogues.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace ibl {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// Warp-uniform copy of a value that every lane of the (converged) warp holds.  REDUX writes a UNIFORM register, so the
// compiler keeps everything derived from the result on the uniform datapath; a value that came from a shared-memory
// load or a special register is per-thread as far as it knows, and each TMA instruction fed from it is wrapped in
// an ELECT / R2UR.BROADCAST loop.
__device__ __forceinline__ uint32_t warp_uniform(uint32_t v) { return __reduce_or_sync(0xffffffffu, v); }

// One lane of the converged warp (elect.sync).  ptxas knows that exactly one thread runs the guarded block and emits the
// TMA instructions inside it back to back; behind `if (lane == 0)` it cannot know, and wraps EVERY such instruction in
// an ELECT / PLOP3 / BRA.U.ANY loop over the "possibly several" active threads.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// for a converged warp: lane 0 polls, the warp re-converges behind it (the polling loop is a divergent exit as far as
// the compiler knows; without the re-convergence point everything after it is per-thread code)
__device__ __forceinline__ void mbar_wait_warp(uint64_t* bar, uint32_t parity) {
  if ((threadIdx.x & 31) == 0) mbar_wait(bar, parity);
  __syncwarp();
}
// the same on a shared-space address (MMA-issuer warps keep barrier addresses as warp-uniform integers)
__device__ __forceinline__ void mbar_wait_warp_a(uint32_t bar_addr, uint32_t parity) {
  if ((threadIdx.x & 31) == 0) {
    uint32_t ok;
    do {
      asm volatile(
          "{\n\t"
          ".reg .pred p;\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
          "selp.u32 %0, 1, 0, p;\n\t"
          "}"
          : "=r"(ok)
          : "r"(bar_addr), "r"(parity)
          : "memory");
    } while (!ok);
  }
  __syncwarp();
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA tiled loads ------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---- the same on shared-space addresses (producer warps that keep ring addresses as warp-uniform integers) --------
__device__ __forceinline__ void mbar_arrive_expect_tx_a(uint32_t bar_addr, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_addr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d_a(uint32_t dst, const CUtensorMap* m, uint32_t bar_addr, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_addr), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d_a(uint32_t dst, const CUtensorMap* m, uint32_t bar_addr, int c0, int c1,
                                              int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_addr), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d_a(uint32_t dst, const CUtensorMap* m, uint32_t bar_addr, int c0, int c1,
                                              int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_addr), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// ---- clusters of two CTAs ("SM pairs"): TMA multicast and cross-CTA barrier arrivals ------------------------------
// 2D tiled load delivered to every CTA of the cluster whose bit is set in `mask` (same smem offset and same mbarrier
// offset in each destination CTA)
__device__ __forceinline__ void tma_load_2d_mc_a(uint32_t dst, const CUtensorMap* m, uint32_t bar_addr, int c0, int c1,
                                                 uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5}], [%2], %3;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_addr), "h"(mask), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d_mc_a(uint32_t dst, const CUtensorMap* m, uint32_t bar_addr, int c0, int c1,
                                                 int c2, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6}], [%2], %3;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar_addr), "h"(mask), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
// arrive on the barrier at this shared::cluster address (another CTA's barrier)
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}

// fire-and-forget: bring one box into L2
__device__ __forceinline__ void tma_prefetch_3d(const CUtensorMap* m, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global [%0, {%1, %2, %3}];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

// ---- warpgroup MMA ------------------------------------------------------------------------------
// Shared-memory matrix descriptor (sm_90 GMMA), K-major operand, 128-byte swizzle: rows of 128 bytes (64 bf16), 8-row
// swizzle atoms 1024 bytes apart.  Advancing the start address by 32 bytes (+2 in 16-byte units) steps 16 elements
// along K inside the swizzled row.
__device__ __forceinline__ uint64_t gmma_desc_kmajor_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fffu);      // start address  [0,14)
  d |= (uint64_t)1 << 16;                           // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024u >> 4) << 32;                // stride byte offset [32,46)
  d |= (uint64_t)1 << 62;                           // layout type: SWIZZLE_128B
  return d;
}
// K-major operand, 64-byte swizzle: rows of 64 bytes (32 bf16, a K = 32 operand without padding), 16-byte chunk j of
// row r stored at chunk position j ^ ((r >> 1) & 3), 8-row atoms 512 bytes apart.  +2 steps 16 elements along K.
__device__ __forceinline__ uint64_t gmma_desc_kmajor_sw64(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fffu);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(512u >> 4) << 32;
  d |= (uint64_t)2 << 62;                           // layout type: SWIZZLE_64B
  return d;
}
// MN-major operand, 128-byte swizzle: rows (K index) of 64 elements = 128 B, 8-row atoms 1024 B apart (SBO); further
// 64-element blocks along M/N are `lbo_bytes` apart (LBO).  16 K rows (one k16 step) are 2048 bytes.
__device__ __forceinline__ uint64_t gmma_desc_mnmajor_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3fffu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= (uint64_t)(1024u >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// Register A operand of one k16 step (WgmmaRS) out of a K-major SW128 tile (128-byte rows, 1024-byte aligned base):
// ldmatrix.x4, lane l addressing tile row `row` at k (16 k16 + 8 (l >> 4)): matrices 0-3 are the fragment's rows 0-7
// and 8-15 at k + 0 and k + 8, so lanes 0-7 / 8-15 / 16-23 / 24-31 name the rows of matrix 0 / 1 / 2 / 3.
__device__ __forceinline__ void ldsm_a_sw128(uint32_t (&r)[4], uint32_t tile, int row, int k16) {
  const uint32_t chunk = (uint32_t)(2 * k16 + ((threadIdx.x >> 4) & 1)) ^ (uint32_t)(row & 7);
  const uint32_t addr = tile + (uint32_t)row * 128u + (chunk << 4);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// named barrier of one consumer warpgroup: id 1 for threads 0..127 of the single-consumer kernels; kernels with two
// consumer warpgroups give each its own id so that one can run its epilogue while the other issues MMAs
__device__ __forceinline__ void wg_sync(int id = 1) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// Hand registers between the warpgroups of a warp-specialised CTA (every warp of the warpgroup executes it): the
// producer gives up what its TMA loop does not need, the MMA warpgroups take it for their accumulators.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// A 128 x N fp32 accumulator held by one warpgroup as two m64 fragments: h[0] = rows 0-63, h[1] = rows 64-127.
// In fragment h, thread t (warp w = t / 32, lane l) holds for every 8-column block i the elements
//   [4i]   (16w + l/4,     8i + 2(l%4))   [4i+1] (same row, column + 1)
//   [4i+2] (16w + l/4 + 8, 8i + 2(l%4))   [4i+3] (same row, column + 1).
template <int N>
struct Acc128 {
  float h[2][N / 2];
  // d += A . B^T over one k16 step; a0 / a1 describe rows 0-63 / 64-127 of A
  template <bool F16 = false, int TA = 0, int TB = 0>
  __device__ __forceinline__ void mma(uint64_t a0, uint64_t a1, uint64_t b, uint32_t accumulate) {
    Wgmma<N, F16, TA, TB>::mma(h[0], a0, b, accumulate);
    Wgmma<N, F16, TA, TB>::mma(h[1], a1, b, accumulate);
  }
  // keeps the compiler from moving accumulator accesses across the asynchronous MMAs
  __device__ __forceinline__ void fence_operands() {
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < N / 2; ++i) asm volatile("" : "+f"(h[j][i])::"memory");
  }
  // Row-per-thread view of 32 accumulator columns [32 ch, 32 ch + 32): thread t of the warpgroup receives row t.
  // The fragments go through `stg` (128 rows x ACC_STG_PITCH floats of shared memory); every thread of the warpgroup
  // must call this with the same ch and the warpgroup's named barrier `bar`.
  __device__ __forceinline__ void rows32(int ch, float* stg, uint32_t (&raw)[32], int bar = 1) const;
};
constexpr int ACC_STG_PITCH = 36;                          // 144-byte rows: conflict-free 16-byte row reads
constexpr int ACC_STG_BYTES = 128 * ACC_STG_PITCH * 4;

template <int N>
__device__ __forceinline__ void Acc128<N>::rows32(int ch, float* stg, uint32_t (&raw)[32], int bar) const {
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  wg_sync(bar);                                            // the previous chunk's reads are done
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = 64 * j + 16 * w + (l >> 2), c = 8 * i + 2 * (l & 3);
      const float* f = &h[j][4 * (4 * ch + i)];
      *reinterpret_cast<float2*>(stg + r * ACC_STG_PITCH + c) = make_float2(f[0], f[1]);
      *reinterpret_cast<float2*>(stg + (r + 8) * ACC_STG_PITCH + c) = make_float2(f[2], f[3]);
    }
  wg_sync(bar);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = *reinterpret_cast<const float4*>(stg + t * ACC_STG_PITCH + 4 * i);
    raw[4 * i] = __float_as_uint(v.x); raw[4 * i + 1] = __float_as_uint(v.y);
    raw[4 * i + 2] = __float_as_uint(v.z); raw[4 * i + 3] = __float_as_uint(v.w);
  }
}

// ---- host: TMA descriptor encoding through the driver entry point (no libcuda link) -----------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_tiled();

// rank-`rank` tiled map with 128B swizzle; dims/strides innermost first (strides in bytes for
// dims 1..rank-1).
int make_tmap(CUtensorMap* out, CUtensorMapDataType dt, int rank, const void* base,
              const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes = 128);

}  // namespace tc
}  // namespace ibl
