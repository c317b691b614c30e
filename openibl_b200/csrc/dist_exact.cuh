// Device helpers shared by the distance paths that screen on the tensor cores and decide in exact fp32
// (tc_dist1.cu: retrieval top-k; rerank.cu: the neighbour pass of k-reciprocal re-ranking).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ibl {

// fp32 -> uint32 whose unsigned order is the float order (and back)
__device__ __forceinline__ uint32_t d1_ord(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float d1_unord(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// exact distance of query row (staged at qrow) and database row ci, one warp; same arithmetic as round 1's
// rescore_sort_kernel: lane-strided float4 FMAs, xor-shuffle tree, fmaf(-2, dot, |q|^2 + |d|^2)
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
