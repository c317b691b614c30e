// Device primitives of every ranking result (include/iblb200.h): ascending by distance, ties to the lowest index,
// padding (+inf, -1).  A rank key is a u64 whose high word is the fp32 distance mapped to an unsigned value of the
// same order and whose low word is the column, so one unsigned compare gives that order.  Also the exact fp32 distance
// and the screening bound shared by the paths that screen on the tensor cores and decide in exact fp32 (tc_gemm.cu,
// tc_dist1.cu: retrieval top-k; rerank.cu: the neighbour pass of k-reciprocal re-ranking).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ibl {

// fp32 -> uint32 whose unsigned order is the float order (and back)
__device__ __forceinline__ uint32_t ord_key(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unord_key(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// (dist, col) -> rank key; ~0ull is the empty key
__device__ __forceinline__ unsigned long long rank_key(float dist, unsigned col) {
  return ((unsigned long long)ord_key(dist) << 32) | col;
}

// out_dist[at], out_idx[at] = the key's distance and idx_base + column, or (+inf, -1) for the empty key
__device__ __forceinline__ void store_ranked(unsigned long long key, long long idx_base, float* out_dist,
                                             long long* out_idx, long long at) {
  if (key == ~0ull) {
    out_dist[at] = INFINITY;
    out_idx[at] = -1;
  } else {
    out_dist[at] = unord_key((uint32_t)(key >> 32));
    out_idx[at] = idx_base + (long long)(uint32_t)(key & 0xffffffffu);
  }
}

// In-place ascending bitonic sort of n (a power of two) keys in shared memory, any block size; barriers before every
// step and after the last, so every thread of the block must call it.
template <typename T>
__device__ void block_bitonic_sort(T* buf, int n) {
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const T a = buf[lo], b = buf[hi];
        if ((a > b) == up) { buf[lo] = b; buf[hi] = a; }
      }
    }
  }
  __syncthreads();
}

// Running top-16 of one row in registers, ascending: (d, col) goes in if it beats td[15].  Sorted insert without a
// dependency chain: the slot is counted with 16 independent compares and every entry is rewritten from the OLD values
// of itself and its left neighbour (descending s).  Constant indices only, so td/ti stay in registers.
__device__ __forceinline__ void top16_insert(float (&td)[16], int (&ti)[16], float d, int col) {
  if (d < td[15]) {
    int pos = 0;
#pragma unroll
    for (int s = 0; s < 16; ++s) pos += (td[s] <= d) ? 1 : 0;
#pragma unroll
    for (int s = 15; s > 0; --s) {
      const bool shift = s > pos, here = s == pos;
      td[s] = shift ? td[s - 1] : (here ? d : td[s]);
      ti[s] = shift ? ti[s - 1] : (here ? col : ti[s]);
    }
    if (pos == 0) { td[0] = d; ti[0] = col; }
  }
}

// exact distance of query row (staged at qrow) and database row ci, one warp: lane-strided float4 FMAs, xor-shuffle
// tree, fmaf(-2, dot, |q|^2 + |d|^2)
__device__ __forceinline__ float d1_exact(const float* qrow, const float* __restrict__ dp, int d, int lane, float an,
                                          float bn) {
  float acc = 0.f;
  for (int i = lane * 4; i < d; i += 128) {
    const float4 a = *reinterpret_cast<const float4*>(qrow + i);
    const float4 b = __ldg(reinterpret_cast<const float4*>(dp + i));
    acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
    acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return fmaf(-2.f, acc, an + bn);
}

// The guard's B: how far a screened distance can lie from |q|^2 + |d|^2 - 2 q.d (the same fp32 norms).  Write
// x = op(x) + r, op = what the MMA reads (the scaled fp16 plane, or bf16 hi + lo with the lo.lo product dropped).
//   operand rounding, rigorous (Cauchy-Schwarz, per pair, the database side by its maximum over the rows):
//       |q.d - screened dot| <= |lo_q| |lo_d| + |q| |r_d| + |r_q| |d| + |r_q| |r_d|
//   fp32 accumulation in the tensor core, STATISTICAL (modelled, not bounded): kappa = 8 sigma of a random walk of
//       one 2^-24 rounding per accumulator update (one per MMA and 16-wide K step), relative to the product
//       magnitudes (|q| + |lo_q| + |r_q|)(max|d| + max|lo_d| + max|r_d|);
//   the epilogue's fma: 2^-23 (|q|^2 + max|d|^2); distance = -2 dot; (1 + d 2^-23) for the fp32 evaluation of B.
// tests/test_host_screening.py mirrors this function and checks the operand part against emulated rounding.
#define D1_ACC_KAPPA 8.f
__device__ __forceinline__ float d1_screen_bound(float q_sq, float q_lo, float q_res, float db_sq_max, float db_lo_max,
                                                 float db_res_max, int d, int mmas_per_k16) {
  const float nq = sqrtf(q_sq), dm = sqrtf(db_sq_max);
  const float dot = q_lo * db_lo_max + nq * db_res_max + q_res * dm + q_res * db_res_max;
  const float acc = D1_ACC_KAPPA * 5.9604645e-8f * sqrtf((float)(d / 16) * mmas_per_k16) * (nq + q_lo + q_res) *
                    (dm + db_lo_max + db_res_max);
  return (2.f * (dot + acc) + 1.1920929e-7f * (q_sq + db_sq_max)) * (1.f + (float)d * 1.1920929e-7f);
}

}  // namespace ibl
