// Fused NetVLAD on the Hopper tensor cores (wgmma), plus a micro-test of its "TN" building block:
// C[m,n] = sum_k A[k,m] B[k,n] with operands MN-major in shared memory (the reduction index is the
// row index), i.e. the layout a TMA box [rows = k][64 contiguous elements] produces.  This is what the
// second NetVLAD contraction needs: vlad[c,k] = sum_s x^[s,c] a[s,k] reads the same [pixel][channel]
// tile the first contraction (logits = x^ W^T, K-major) already staged, so the feature map is read
// from HBM once.
#include "common.cuh"
#include "tc_common.cuh"

namespace ibl {

using namespace tc;

// ---- micro-test: one CTA, M = 128, N = 64, K = 128, bf16x3 -----------------------------------------
__global__ void __launch_bounds__(128, 1)
tn_gemm_test_kernel(const __grid_constant__ CUtensorMap tm_ahi, const __grid_constant__ CUtensorMap tm_alo,
                    const __grid_constant__ CUtensorMap tm_bhi, const __grid_constant__ CUtensorMap tm_blo,
                    float* __restrict__ C) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // A_hi: two [128 k][64 m] blocks (32 KB), A_lo (32 KB), B_hi [128 k][64 n] (16 KB), B_lo (16 KB)
  uint8_t* a_hi = smem;
  uint8_t* a_lo = smem + 32768;
  uint8_t* b_hi = smem + 65536;
  uint8_t* b_lo = smem + 81920;
  float* stg = reinterpret_cast<float*>(smem + 98304);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 98304 + ACC_STG_BYTES);
  if (threadIdx.x == 0) {
    mbar_init(&bars[0], 1);
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bars[0], 98304);
    tma_load_2d(a_hi, &tm_ahi, &bars[0], 0, 0);
    tma_load_2d(a_hi + 16384, &tm_ahi, &bars[0], 64, 0);
    tma_load_2d(a_lo, &tm_alo, &bars[0], 0, 0);
    tma_load_2d(a_lo + 16384, &tm_alo, &bars[0], 64, 0);
    tma_load_2d(b_hi, &tm_bhi, &bars[0], 0, 0);
    tma_load_2d(b_lo, &tm_blo, &bars[0], 0, 0);
  }
  mbar_wait(&bars[0], 0);
  Acc128<64> acc;
  wgmma_fence();
  for (int ks = 0; ks < 8; ++ks) {   // 16 k-rows (2048 B) per MMA
    const uint32_t off = ks * 2048;
    const uint64_t dah0 = gmma_desc_mnmajor_sw128(smem_u32(a_hi) + off, 16384);
    const uint64_t dah1 = gmma_desc_mnmajor_sw128(smem_u32(a_hi) + 16384 + off, 16384);
    const uint64_t dal0 = gmma_desc_mnmajor_sw128(smem_u32(a_lo) + off, 16384);
    const uint64_t dal1 = gmma_desc_mnmajor_sw128(smem_u32(a_lo) + 16384 + off, 16384);
    const uint64_t dbh = gmma_desc_mnmajor_sw128(smem_u32(b_hi) + off, 0);
    const uint64_t dbl = gmma_desc_mnmajor_sw128(smem_u32(b_lo) + off, 0);
    acc.mma<false, 1, 1>(dal0, dal1, dbh, ks > 0 ? 1u : 0u);
    acc.mma<false, 1, 1>(dah0, dah1, dbl, 1u);
    acc.mma<false, 1, 1>(dah0, dah1, dbh, 1u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  acc.fence_operands();
  const int m = threadIdx.x;
#pragma unroll
  for (int ch = 0; ch < 2; ++ch) {
    uint32_t raw[32];
    acc.rows32(ch, stg, raw);
#pragma unroll
    for (int j = 0; j < 32; ++j) C[m * 64 + ch * 32 + j] = __uint_as_float(raw[j]);
  }
}

// A [128 k][128 m] fp32, B [128 k][64 n] fp32 (device) -> C [128 m][64 n] = A^T B
int debug_gemm_tn(const float* A, const float* B, float* C, cudaStream_t s) {
  __nv_bfloat16 *pa = nullptr, *pb = nullptr;
  IBL_CUDA_OK(cudaMalloc(&pa, 128 * 128 * 2 * 2));
  IBL_CUDA_OK(cudaMalloc(&pb, 128 * 64 * 2 * 2));
  int rc = launch_f32_to_planes(A, 128 * 128, pa, pa + 128 * 128, s);
  if (rc == IBL_OK) rc = launch_f32_to_planes(B, 128 * 64, pb, pb + 128 * 64, s);
  CUtensorMap maps[4];
  uint64_t da[2] = {128, 128}, db[2] = {64, 128}, sa[1] = {128 * 2}, sb[1] = {64 * 2};
  uint32_t box[2] = {64, 128};
  if (rc == IBL_OK) rc = make_tmap(&maps[0], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, pa, da, sa, box);
  if (rc == IBL_OK) rc = make_tmap(&maps[1], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, pa + 128 * 128, da, sa, box);
  if (rc == IBL_OK) rc = make_tmap(&maps[2], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, pb, db, sb, box);
  if (rc == IBL_OK) rc = make_tmap(&maps[3], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, pb + 128 * 64, db, sb, box);
  if (rc == IBL_OK) {
    const int smem = 98304 + ACC_STG_BYTES + 1024 + 64;
    cudaFuncSetAttribute(tn_gemm_test_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    tn_gemm_test_kernel<<<1, 128, smem, s>>>(maps[0], maps[1], maps[2], maps[3], C);
    if (cudaGetLastError() != cudaSuccess) rc = IBL_ERR_CUDA;
  }
  cudaError_t ce = cudaStreamSynchronize(s);
  cudaFree(pa);
  cudaFree(pb);
  if (rc == IBL_OK && ce != cudaSuccess) { set_last_error(cudaGetErrorString(ce)); rc = IBL_ERR_CUDA; }
  return rc;
}

// =====================================================================================================
// Fused NetVLAD (reference ibl/models/netvlad.py:44-61 + the intra-normalisation / L2 of :78-80)
//
//   x^[s,:] = x[s,:] / max(|x[s,:]|, eps)                       |x[s,:]|^2 comes from the conv5_3 epilogue
//   z[s,k]  = W[k,:] . x^[s,:]          GEMM 1 (wgmma, K-major operands: pixel tile x channel chunk)
//   a[s,:]  = softmax_k z[s,:]          one pixel per thread, fp32, max-subtracted
//   V[c,k]  = sum_s x^[s,c] a[s,k]      GEMM 2 (wgmma, MN-major operands: the SAME [pixel][channel]
//                                       tiles, and a' = a/|x| written to shared memory by the softmax)
//   vlad[k,c] = V[c,k] - cent[k,c] * sum_s a[s,k]
//
// K <= 64 clusters run on the K = 64 layout: rows K..63 of the W planes are zero and their logits are set to -inf
// before the softmax, so their a, a', sum_s a and V columns are exactly 0.  The partials keep 64 rows; only the
// finalisation knows K (it reads centroid rows k < K and writes [B][K][512]).
//
// One work unit = (image, every G-th 128-pixel tile); a unit accumulates V (512 x 64 fp32, too large for the
// registers of one warpgroup) in its own partial slice in global memory, which stays in L2: every element is
// read-modified-written by the same thread, tile after tile, in tile order.  ONE LAUNCH: the unit that arrives last for an image
// (atomic ticket in global memory) adds the G partials in index order (L2 hits), subtracts the centroid term
// and applies the intra-normalisation and the global L2 (netvlad.py:78-80) before the kernel ends -- there is
// no finalize kernel.  G depends on S only, never on the batch, so an image's descriptor is bit-identical
// whatever batch it travels in.  The feature map is read from HBM once (the second pass over a tile's
// channel chunks hits L2).  Both contractions are bf16x3.
//
// Warp roles: warps 0-3 consumer warpgroup (GEMM 1, softmax, GEMM 2, unit epilogue), warp 4 TMA producer.
// Shared memory: 3 stages of 64 KiB (GEMM 1 stage: X_hi | X_lo | W_hi,W_lo of one 64-channel chunk;
// GEMM 2 stage: X_hi c0 | X_hi c1 | X_lo c0 | X_lo c1 of one 128-channel block) + a' hi/lo (32 KiB)
// + the accumulator transposition buffer.
// =====================================================================================================
struct NvTcArgs {
  int B, S, G, T;                 // images, pixels per image, units per image, 128-pixel tiles per image
  int K;                          // clusters, 1..64
  int ssq_parts;                  // number of partial |x|^2 planes to add
  const float* ssq;               // [ssq_parts][B*S]
  int normalize_input;
  float* part;                    // [B*G][64][512]   partial V^T (k-major rows, c contiguous)
  float* asum_part;               // [B*G][64]
  const float* cent;              // [K][512] centroids
  float* vlad_raw;                // [B][K][512] un-normalised VLAD (nullable)
  float* vlad_norm;               // [B][K*512] intra-normalised + L2-normalised descriptor (nullable)
  int* ticket;                    // [B] zero on entry; the unit that takes ticket G-1 finalises the image and resets it
};

constexpr int NV_STAGE = 65536, NV_NSTAGE = 3, NV_SLOT = 16384;

// The CTA's tiles in processing order: units blockIdx.x, +gridDim.x, ...; inside a unit tiles g, g+G, ...
struct NvIter {
  int u, t, useq, G, T, n_units, stride;
  __device__ void init(int first_unit, int stride_, int G_, int T_, int n_units_) {
    G = G_; T = T_; n_units = n_units_; stride = stride_;
    u = first_unit; useq = 0; t = u % G;
  }
  __device__ bool valid() const { return u < n_units; }
  __device__ bool first() const { return t < G; }
  __device__ bool last() const { return t + G >= T; }
  __device__ void next() {
    t += G;
    if (t >= T) { u += stride; ++useq; t = u % G; }
  }
};

// Finalisation of image b by the consumer warpgroup (128 threads) of the unit that arrived last:
//   vlad[k,c] = sum_g part[b,g,k,c] - cent[k,c] * sum_g asum[b,g,k]   (partials added in index order: deterministic)
//   intra-normalise every cluster row (netvlad.py:78), flatten k-major, global L2 (:79-80).
// Warp q owns rows q*16 .. q*16+15, lane L the channels L, L+32, ...; every thread rescales exactly the elements it
// wrote itself, so the second pass needs no fence.  `sm` is the 260-float asum scratch of the kernel.  Rows k >= K are
// zero in the partials: they are neither read from the centroids nor written, and add nothing to the norms.
__device__ __forceinline__ void nv_finalize_image(const NvTcArgs& a, int b, int q, int lane, float* sm) {
  const int tid = q * 32 + lane;
  const int K = a.K;
  const long long ub = (long long)b * a.G;
  if (tid < 64) {
    float s = 0.f;
    for (int g = 0; g < a.G; ++g) s += __ldcg(a.asum_part + (ub + g) * 64 + tid);
    sm[tid] = s;
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");
  float tot = 0.f;
  // Latency-bound on one SM (640 KB from L2): two rows per iteration, 16-byte loads, all 2 x 4 x (G + 1) loads of an
  // iteration issued before the first add.  Lane L owns channels 4L .. 4L+3 of every 128-channel block.
#pragma unroll 1
  for (int r = 0; r < 16; r += 2) {
    float4 v[2][4], cz[2][4];
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[u][j] = make_float4(0.f, 0.f, 0.f, 0.f);
        cz[u][j] = q * 16 + r + u < K
                       ? __ldg(reinterpret_cast<const float4*>(a.cent + (q * 16 + r + u) * 512 + 4 * lane + 128 * j))
                       : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
    for (int g = 0; g < 4; ++g) {                      // G <= 4 (netvlad_tc_units); partials added in index order
      if (g < a.G) {
        float4 t[2][4];
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
          for (int j = 0; j < 4; ++j)
            t[u][j] = __ldcg(reinterpret_cast<const float4*>(a.part + ((ub + g) * 64 + q * 16 + r + u) * 512 + 4 * lane + 128 * j));
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            v[u][j].x += t[u][j].x; v[u][j].y += t[u][j].y; v[u][j].z += t[u][j].z; v[u][j].w += t[u][j].w;
          }
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int k = q * 16 + r + u;
      const float asum = sm[k];
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[u][j].x -= cz[u][j].x * asum; v[u][j].y -= cz[u][j].y * asum;
        v[u][j].z -= cz[u][j].z * asum; v[u][j].w -= cz[u][j].w * asum;
        ss = fmaf(v[u][j].x, v[u][j].x, ss); ss = fmaf(v[u][j].y, v[u][j].y, ss);
        ss = fmaf(v[u][j].z, v[u][j].z, ss); ss = fmaf(v[u][j].w, v[u][j].w, ss);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
      float s2 = 0.f;
      const long long row = ((long long)b * K + k) * 512 + 4 * lane;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (a.vlad_raw && k < K) *reinterpret_cast<float4*>(a.vlad_raw + row + 128 * j) = v[u][j];
        const float4 w = make_float4(v[u][j].x * inv, v[u][j].y * inv, v[u][j].z * inv, v[u][j].w * inv);
        s2 = fmaf(w.x, w.x, s2); s2 = fmaf(w.y, w.y, s2); s2 = fmaf(w.z, w.z, s2); s2 = fmaf(w.w, w.w, s2);
        if (a.vlad_norm && k < K) *reinterpret_cast<float4*>(a.vlad_norm + row + 128 * j) = w;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      tot += s2;
    }
  }
  if (!a.vlad_norm) return;                          // block-uniform
  if (lane == 0) sm[128 + q] = tot;
  asm volatile("bar.sync 1, 128;" ::: "memory");
  const float ginv = 1.f / fmaxf(sqrtf((sm[128] + sm[129]) + (sm[130] + sm[131])), 1e-12f);
#pragma unroll 1
  for (int r8 = 0; r8 < 2; ++r8) {                   // 8 rows = 32 independent 16-byte loads per thread in flight
    const int k0 = q * 16 + r8 * 8;
    float4* o = reinterpret_cast<float4*>(a.vlad_norm + ((long long)b * K + k0) * 512 + 4 * lane);
    if (k0 + 8 <= K) {                               // warp-uniform: 8 whole rows
      float4 t[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) t[i] = o[(i >> 2) * 128 + 32 * (i & 3)];
#pragma unroll
      for (int i = 0; i < 32; ++i)
        o[(i >> 2) * 128 + 32 * (i & 3)] = make_float4(t[i].x * ginv, t[i].y * ginv, t[i].z * ginv, t[i].w * ginv);
    } else {                                         // the 8-row block that K < 64 cuts: its rows below K only
#pragma unroll 1
      for (int r = 0; k0 + r < K; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float4 t = o[r * 128 + 32 * j];
          o[r * 128 + 32 * j] = make_float4(t.x * ginv, t.y * ginv, t.z * ginv, t.w * ginv);
        }
    }
  }
}

__global__ void __launch_bounds__(160, 1)
netvlad_tc_kernel(const __grid_constant__ CUtensorMap tm_xhi, const __grid_constant__ CUtensorMap tm_xlo,
                  const __grid_constant__ CUtensorMap tm_whi, const __grid_constant__ CUtensorMap tm_wlo,
                  const NvTcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* asm_hi = smem + NV_NSTAGE * NV_STAGE;
  uint8_t* asm_lo = asm_hi + NV_SLOT;
  // the accumulator transposition of the logits runs while a' is free (GEMM 2 of the previous tile has retired, the
  // softmax has not written yet): it borrows the a' buffers
  float* stg = reinterpret_cast<float*>(asm_hi);
  static_assert(ACC_STG_BYTES <= 2 * NV_SLOT, "transposition buffer inside a' hi | lo");
  uint64_t* bars = reinterpret_cast<uint64_t*>(asm_lo + NV_SLOT);
  uint64_t* full_bar = bars;                 // [3]
  uint64_t* empty_bar = bars + 3;            // [3] one arrival per consumer warp
  float* asum_sm = reinterpret_cast<float*>(bars + 16);   // [4 warps][64]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tm_xhi); tma_prefetch_desc(&tm_xlo); tma_prefetch_desc(&tm_whi); tma_prefetch_desc(&tm_wlo);
    for (int i = 0; i < 3; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();
  const int n_units = a.B * a.G;

  if (warp == 4) {
    // TMA producer: convergent warp, one elected lane issues, warp-uniform operands.  Per tile: the 8 GEMM 1 stages,
    // then the 4 GEMM 2 stages (L2 hits), in the order the consumer walks them.
    const uint32_t smem_a = warp_uniform(smem_u32(smem));
    const uint32_t bars_a = smem_a + NV_NSTAGE * NV_STAGE + 2 * NV_SLOT;
    const uint32_t full_a = bars_a, empty_a = bars_a + 24;
    int stage = 0; uint32_t phase = 0;
    NvIter c1;
    c1.init(blockIdx.x, gridDim.x, a.G, a.T, n_units);
    while (c1.valid()) {
      const int b = (int)warp_uniform((uint32_t)(c1.u / a.G)), p0 = (int)warp_uniform((uint32_t)(c1.t * 128));
      for (int c = 0; c < 8; ++c) {           // GEMM 1 stages: one 64-channel chunk + its W chunk
        const uint32_t sg = warp_uniform((uint32_t)stage);
        mbar_wait_warp_a(empty_a + 8 * sg, phase ^ 1);
        const uint32_t st = smem_a + sg * NV_STAGE, fb = full_a + 8 * sg;
        if (elect_one()) {
          mbar_arrive_expect_tx_a(fb, 3 * NV_SLOT);
          tma_load_3d_a(st, &tm_xhi, fb, c * 64, p0, b);
          tma_load_3d_a(st + NV_SLOT, &tm_xlo, fb, c * 64, p0, b);
          tma_load_2d_a(st + 2 * NV_SLOT, &tm_whi, fb, c * 64, 0);
          tma_load_2d_a(st + 2 * NV_SLOT + 8192, &tm_wlo, fb, c * 64, 0);
        }
        __syncwarp();
        if (++stage == NV_NSTAGE) { stage = 0; phase ^= 1; }
      }
      for (int cb = 0; cb < 4; ++cb) {        // GEMM 2 stages: one 128-channel block
        const uint32_t sg = warp_uniform((uint32_t)stage);
        mbar_wait_warp_a(empty_a + 8 * sg, phase ^ 1);
        const uint32_t st = smem_a + sg * NV_STAGE, fb = full_a + 8 * sg;
        if (elect_one()) {
          mbar_arrive_expect_tx_a(fb, 4 * NV_SLOT);
          tma_load_3d_a(st, &tm_xhi, fb, cb * 128, p0, b);
          tma_load_3d_a(st + NV_SLOT, &tm_xhi, fb, cb * 128 + 64, p0, b);
          tma_load_3d_a(st + 2 * NV_SLOT, &tm_xlo, fb, cb * 128, p0, b);
          tma_load_3d_a(st + 3 * NV_SLOT, &tm_xlo, fb, cb * 128 + 64, p0, b);
        }
        __syncwarp();
        if (++stage == NV_NSTAGE) { stage = 0; phase ^= 1; }
      }
      c1.next();
      if (c1.valid()) {                       // rolling L2 prefetch: the NEXT tile's boxes, behind this tile's loads
        const int bn = (int)warp_uniform((uint32_t)(c1.u / a.G));
        const int pn = (int)warp_uniform((uint32_t)(c1.t * 128));
        if (elect_one()) {
          for (int c2i = 0; c2i < 8; ++c2i) {
            tma_prefetch_3d(&tm_xhi, c2i * 64, pn, bn);
            tma_prefetch_3d(&tm_xlo, c2i * 64, pn, bn);
          }
        }
        __syncwarp();
      }
    }
  } else {
    const int q = warp;
    const int s_loc = threadIdx.x;               // pixel row inside the tile
    const uint32_t smem_a = smem_u32(smem);
    const uint32_t ah = smem_u32(asm_hi), al = smem_u32(asm_lo);
    int stage = 0; uint32_t phase = 0;
    auto release = [&](int st) { if (lane == 0) mbar_arrive(&empty_bar[st]); };
    float as0 = 0.f, as1 = 0.f;                  // sum_s a[s,k] for k = 2*lane, 2*lane+1 (this warp's rows)
    NvIter cur;
    cur.init(blockIdx.x, gridDim.x, a.G, a.T, n_units);
    for (int it = 0; cur.valid(); cur.next(), ++it) {
      const int unit = cur.u, b = unit / a.G;
      float* po = a.part + (long long)unit * 64 * 512;
      {
        const int s = cur.t * 128 + s_loc;
        const bool valid = s < a.S;
        float inv = 1.f;
        if (valid && a.normalize_input) {
          float ss = 0.f;
          for (int p = 0; p < a.ssq_parts; ++p) ss += __ldg(a.ssq + (long long)p * a.B * a.S + (long long)b * a.S + s);
          inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
        }
        // ---- GEMM 1: Z[128 px, 64 clusters] = x . W^T (bf16x3) ----
        float z[64];
        {
          Acc128<64> zacc;
          int prev = -1;
          for (int c = 0; c < 8; ++c) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_a + stage * NV_STAGE;
            const uint64_t xh = gmma_desc_kmajor_sw128(sa), xl = gmma_desc_kmajor_sw128(sa + NV_SLOT);
            const uint64_t wh = gmma_desc_kmajor_sw128(sa + 2 * NV_SLOT);
            const uint64_t wl = gmma_desc_kmajor_sw128(sa + 2 * NV_SLOT + 8192);
            constexpr uint64_t kHalf = 64 * 128 / 16;   // pixel rows 64-127: +8 KiB
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const uint64_t ko = (uint64_t)(k * 2);
              zacc.mma(xl + ko, xl + kHalf + ko, wh + ko, (c > 0 || k > 0) ? 1u : 0u);
              zacc.mma(xh + ko, xh + kHalf + ko, wl + ko, 1u);
              zacc.mma(xh + ko, xh + kHalf + ko, wh + ko, 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (prev >= 0) release(prev);
            prev = stage;
            if (++stage == NV_NSTAGE) { stage = 0; phase ^= 1; }
          }
          wgmma_wait<0>();
          zacc.fence_operands();
          release(prev);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t r0[32];
            zacc.rows32(h, stg, r0);
#pragma unroll
            for (int j = 0; j < 32; ++j) z[h * 32 + j] = __uint_as_float(r0[j]) * inv;
          }
          wg_sync();                                 // every row has read its logits before a' overwrites them
        }
        if (a.K < 64) {                              // padded clusters: assignment exactly 0
#pragma unroll
          for (int j = 0; j < 64; ++j)
            if (j >= a.K) z[j] = -INFINITY;
        }
        float m = z[0];
#pragma unroll
        for (int j = 1; j < 64; ++j) m = fmaxf(m, z[j]);
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 64; ++j) { z[j] = expf(z[j] - m); sum += z[j]; }
        const float rs = valid ? 1.f / sum : 0.f;
#pragma unroll
        for (int j = 0; j < 64; ++j) z[j] *= rs;   // a[s,:] (0 for rows past the image)
        // a' = a * inv as bf16 hi/lo, MN-major SW128 row s_loc: 8 chunks of 8 values, chunk j at j^(s&7)
        {
          uint8_t* rh = asm_hi + s_loc * 128;
          uint8_t* rl = asm_lo + s_loc * 128;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float x0 = z[8 * j + 2 * e] * inv, x1 = z[8 * j + 2 * e + 1] * inv;
              const __nv_bfloat16 h0 = __float2bfloat16_rn(x0), h1 = __float2bfloat16_rn(x1);
              __nv_bfloat162 hh(h0, h1);
              __nv_bfloat162 ll = __floats2bfloat162_rn(x0 - __bfloat162float(h0), x1 - __bfloat162float(h1));
              hi[e] = *reinterpret_cast<uint32_t*>(&hh);
              lo[e] = *reinterpret_cast<uint32_t*>(&ll);
            }
            const int pos = (j ^ (s_loc & 7)) * 16;
            *reinterpret_cast<uint4*>(rh + pos) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            *reinterpret_cast<uint4*>(rl + pos) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
          }
        }
        fence_proxy_async();                       // generic-proxy smem writes -> visible to the tensor core
        wg_sync();                                 // every row of a' is written
        // column sums of a over this warp's 32 rows: butterfly, lane L ends with columns 2L, 2L+1
        {
          float w32[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const float keep = (lane & 16) ? z[32 + i] : z[i];
            const float send = (lane & 16) ? z[i] : z[32 + i];
            w32[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
          }
          float w16[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float keep = (lane & 8) ? w32[16 + i] : w32[i];
            const float send = (lane & 8) ? w32[i] : w32[16 + i];
            w16[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
          }
          float w8[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float keep = (lane & 4) ? w16[8 + i] : w16[i];
            const float send = (lane & 4) ? w16[i] : w16[8 + i];
            w8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
          }
          float w4[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float keep = (lane & 2) ? w8[4 + i] : w8[i];
            const float send = (lane & 2) ? w8[i] : w8[4 + i];
            w4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
          }
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float keep = (lane & 1) ? w4[2 + i] : w4[i];
            const float send = (lane & 1) ? w4[i] : w4[2 + i];
            const float v = keep + __shfl_xor_sync(0xffffffffu, send, 1);
            if (i == 0) as0 += v; else as1 += v;
          }
        }
        // ---- GEMM 2: V[128 c, 64 k] (4 channel blocks) += X^T a', added into the unit's partial ----
        const bool fresh = cur.first();
        const int fw = q, fl = lane;
        for (int cb = 0; cb < 4; ++cb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_a + stage * NV_STAGE;
          Acc128<64> v;
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 8; ++ks) {     // 16 pixel rows (2048 B) per MMA
            const uint32_t off = ks * 2048;
            const uint64_t xh0 = gmma_desc_mnmajor_sw128(sa + off, NV_SLOT);
            const uint64_t xh1 = gmma_desc_mnmajor_sw128(sa + NV_SLOT + off, NV_SLOT);
            const uint64_t xl0 = gmma_desc_mnmajor_sw128(sa + 2 * NV_SLOT + off, NV_SLOT);
            const uint64_t xl1 = gmma_desc_mnmajor_sw128(sa + 3 * NV_SLOT + off, NV_SLOT);
            const uint64_t bh = gmma_desc_mnmajor_sw128(ah + off, 0);
            const uint64_t bl = gmma_desc_mnmajor_sw128(al + off, 0);
            v.mma<false, 1, 1>(xl0, xl1, bh, ks > 0 ? 1u : 0u);
            v.mma<false, 1, 1>(xh0, xh1, bl, 1u);
            v.mma<false, 1, 1>(xh0, xh1, bh, 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          v.fence_operands();
          release(stage);
          if (++stage == NV_NSTAGE) { stage = 0; phase ^= 1; }
          // fragment element (channel row r, cluster column k) -> part[k][cb*128 + r]
#pragma unroll
          for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int r = 64 * j + 16 * fw + (fl >> 2) + ((e & 2) ? 8 : 0);
                const int k = 8 * i + 2 * (fl & 3) + (e & 1);
                float* dst = po + (long long)k * 512 + cb * 128 + r;
                *dst = fresh ? v.h[j][4 * i + e] : *dst + v.h[j][4 * i + e];
              }
        }
      }
      if (cur.last()) {
        // ---- unit epilogue: partial sum_s a, then the last unit of the image finalises it ----
        asum_sm[q * 64 + 2 * lane] = as0;
        asum_sm[q * 64 + 2 * lane + 1] = as1;
        wg_sync();
        if (threadIdx.x < 64) {
          const int k = threadIdx.x;
          a.asum_part[(long long)unit * 64 + k] = asum_sm[k] + asum_sm[64 + k] + asum_sm[128 + k] + asum_sm[192 + k];
        }
        // ---- last unit of the image finalises it (threadfence-reduction pattern) ----
        __threadfence();                             // this thread's partial is visible device-wide
        wg_sync();
        int* flag_sm = reinterpret_cast<int*>(asum_sm + 256);
        if (threadIdx.x == 0) {
          const int tk = atomicAdd(a.ticket + b, 1);
          const int lastu = (tk == a.G - 1) ? 1 : 0;
          if (lastu) a.ticket[b] = 0;                // self-cleaning: the next launch finds zeros again
          *flag_sm = lastu;
        }
        wg_sync();
        if (*flag_sm) {
          __threadfence();
          nv_finalize_image(a, b, q, lane, asum_sm);
        }
        wg_sync();                                   // flag_sm / asum_sm are reused by the next unit
        as0 = 0.f; as1 = 0.f;
      }
    }
  }
}

// (A 4-CTA-cluster variant that reads every feature byte once -- channels split over the cluster, partial logits
// reduce-scattered and a' all-gathered through DSMEM -- was parity-green but measured 62-77 us against 35 us for
// this kernel and was removed from the product library; see git history, round 1: tc_netvlad4.cu.)
// Units per image: a function of S ONLY (never of the batch), so that an image's partial sums are formed and added
// in the same order whatever batch it is part of -- descriptors are bit-identical across batch compositions and world
// sizes (the 250k gallery ranks identically on 1 and 8 GPUs).  4 units x 32 images = 128 CTAs for the batch-32 step.
int netvlad_tc_units(int B, int S) {
  (void)B;
  const int T = cdiv(S, 128);
  return T < 4 ? T : 4;
}

// x planes [B,S,512] (hi, lo), w planes [64,512] (hi, lo; rows K..63 zero), ssq [parts][B*S], cent [K,512] fp32,
// vlad_raw [B,K,512], vlad_norm [B,K*512]; part / asum_part are sized for 64 clusters whatever K is
int launch_netvlad_tc(const __nv_bfloat16* x_hi, const __nv_bfloat16* x_lo, int B, int S, int K,
                      const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo, const float* ssq, int ssq_parts,
                      const float* cent, bool normalize_input, float* part, float* asum_part, int* ticket,
                      float* vlad_raw, float* vlad_norm, cudaStream_t s) {
  IBL_REQUIRE(K >= 1 && K <= 64, "the tensor-core NetVLAD kernel serves 1..64 clusters");
  CUtensorMap mx_hi, mx_lo, mw_hi, mw_lo;
  {
    uint64_t dims[3] = {512, (uint64_t)S, (uint64_t)B};
    uint64_t str[2] = {512 * 2, (uint64_t)S * 512 * 2};
    uint32_t box[3] = {64, 128, 1};
    IBL_RET(make_tmap(&mx_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, x_hi, dims, str, box));
    IBL_RET(make_tmap(&mx_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, x_lo, dims, str, box));
  }
  {
    uint64_t dims[2] = {512, 64};
    uint64_t str[1] = {512 * 2};
    uint32_t box[2] = {64, 64};
    IBL_RET(make_tmap(&mw_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, w_hi, dims, str, box));
    IBL_RET(make_tmap(&mw_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, w_lo, dims, str, box));
  }
  NvTcArgs a{};
  a.B = B; a.S = S; a.K = K; a.T = cdiv(S, 128); a.G = netvlad_tc_units(B, S);
  a.ssq = ssq; a.ssq_parts = ssq_parts; a.normalize_input = normalize_input ? 1 : 0;
  a.part = part; a.asum_part = asum_part;
  a.cent = cent; a.vlad_raw = vlad_raw; a.vlad_norm = vlad_norm; a.ticket = ticket;
  const int smem = NV_NSTAGE * NV_STAGE + 2 * NV_SLOT + 1024 + 128 + 4 * 64 * 4 + 16;
  static DeviceOnce attr_done;   // the attribute is per device
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(netvlad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_done.mark();
  }
  const int sms = device_sm_count();
  const int units = B * a.G;
  netvlad_tc_kernel<<<units < sms ? units : sms, 160, smem, s>>>(mx_hi, mx_lo, mw_hi, mw_lo, a);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

}  // namespace ibl
