// Backward of the PCA-whitening layer y = v W^T + b (EmbedNetPCA.pca_layer, reference ibl/models/netvlad.py:105-107,
// a 1x1 conv differentiated by autograd there), W [P,D], v [N,D], gy = dL/dy [N,P]:
//
//   dgrad   gv[n,d] = sum_p gy[n,p] W[p,d]     contraction over P: W is read as an MN-major operand, a TMA box of
//                                              [64 p rows][64 contiguous d] of the engine's W planes (the same planes
//                                              the forward reads K-major).  Bound by the weight read: every plane
//                                              element is read once per call for up to 128 batch rows.
//   wgrad   gW[p,d] = sum_n gy[n,p] v[n,d]     contraction over the batch rows: both operands MN-major, the rows
//                                              padded to 16 by the TMA's out-of-bounds zero fill.  Bound by the
//                                              [P,D] fp32 store, written once, coalesced along d.
//   gb[p]   = sum_n gy[n,p]                    a small CUDA-core reduction.
//
// Both GEMMs are one kernel: the accumulator rows are 128 output columns d (A operand = W or v, MN-major), its
// columns BN output rows c (B operand = gy, K-major [rows n][64 p] for dgrad, MN-major [16 rows n][64 p] for wgrad),
// bf16 hi/lo x3 with fp32 accumulation, TMA into an mbarrier ring, one producer warp and one consumer warpgroup.
// The fp32 math mode runs the same contractions on CUDA cores (pca_tn_simt_kernel).
#include "common.cuh"
#include "tc_common.cuh"

namespace ibl {

using namespace tc;

struct PcaBwdArgs {
  int D;          // output columns (the A operand's MN extent)
  int cols;       // output rows: N (dgrad) or P (wgrad)
  int K;          // contraction length: P (dgrad) or N (wgrad)
  int d_tiles, c_tiles;
  float* out;     // [cols][D]
};

// The wgmma fp32 accumulator rounds toward zero on every accumulation (see WG_CHAIN_BOXES in tc_conv_bwd.cu): a chain
// is restarted every PB_CHAIN_ROWS contraction rows and added into the output with ordinary fp32 adds, so a 4096-long
// dgrad contraction is four chains of 192 MMAs.
constexpr int PB_CHAIN_ROWS = 1024;

template <int BN, int TB, int KR>
struct PcaBwdShape {
  static constexpr int A_BOX = KR * 128;                   // [KR rows][64 d] bf16
  static constexpr int B_BYTES = BN * KR * 2;              // one plane of the gy tile
  static constexpr int STAGE = 4 * A_BOX + 2 * B_BYTES;    // A hi d0,d1 | A lo d0,d1 | B hi | B lo
};

template <int BN, int TB, int KR, int STAGES>
__global__ void __launch_bounds__(160, 1)
pca_bwd_tc_kernel(const __grid_constant__ CUtensorMap tm_ahi, const __grid_constant__ CUtensorMap tm_alo,
                  const __grid_constant__ CUtensorMap tm_bhi, const __grid_constant__ CUtensorMap tm_blo,
                  const PcaBwdArgs g) {
  using Sh = PcaBwdShape<BN, TB, KR>;
  constexpr int A_BOX = Sh::A_BOX, B_BYTES = Sh::B_BYTES, STAGE = Sh::STAGE;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* stg = reinterpret_cast<float*>(smem + STAGES * STAGE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE + ACC_STG_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kchunks = (g.K + KR - 1) / KR;
  const int total = g.d_tiles * g.c_tiles;

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tm_ahi); tma_prefetch_desc(&tm_alo); tma_prefetch_desc(&tm_bhi); tma_prefetch_desc(&tm_blo);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp == 4) {
    // producer: convergent warp, one elected lane issues, warp-uniform operands
    const uint32_t smem_a = warp_uniform(smem_u32(smem));
    const uint32_t full_a = smem_a + STAGES * STAGE + ACC_STG_BYTES, empty_a = full_a + 8 * STAGES;
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < total; item += gridDim.x) {
      const int d0 = (int)warp_uniform((uint32_t)((item % g.d_tiles) * 128));
      const int c0 = (int)warp_uniform((uint32_t)((item / g.d_tiles) * BN));
      for (int kc = 0; kc < kchunks; ++kc) {
        const uint32_t sg = warp_uniform((uint32_t)stage);
        mbar_wait_warp_a(empty_a + 8 * sg, phase ^ 1);
        const uint32_t st = smem_a + sg * STAGE, fb = full_a + 8 * sg;
        const int k0 = (int)warp_uniform((uint32_t)(kc * KR));
        if (elect_one()) {
          mbar_arrive_expect_tx_a(fb, STAGE);
          tma_load_2d_a(st, &tm_ahi, fb, d0, k0);
          tma_load_2d_a(st + A_BOX, &tm_ahi, fb, d0 + 64, k0);
          tma_load_2d_a(st + 2 * A_BOX, &tm_alo, fb, d0, k0);
          tma_load_2d_a(st + 3 * A_BOX, &tm_alo, fb, d0 + 64, k0);
          const uint32_t sb = st + 4 * A_BOX;
          if (TB == 0) {            // [BN rows n][64 p]
            tma_load_2d_a(sb, &tm_bhi, fb, k0, c0);
            tma_load_2d_a(sb + B_BYTES, &tm_blo, fb, k0, c0);
          } else {                  // BN / 64 boxes of [KR rows n][64 p]
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) {
              tma_load_2d_a(sb + j * A_BOX, &tm_bhi, fb, c0 + 64 * j, k0);
              tma_load_2d_a(sb + B_BYTES + j * A_BOX, &tm_blo, fb, c0 + 64 * j, k0);
            }
          }
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // consumer warpgroup; in the epilogue thread t owns output column d0 + t of every output row of the tile
    const uint32_t smem_a = smem_u32(smem);
    constexpr int CHAIN = PB_CHAIN_ROWS / KR;
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < total; item += gridDim.x) {
      const int d0 = (item % g.d_tiles) * 128, c0 = (item / g.d_tiles) * BN;
      const int d = d0 + (int)threadIdx.x;
      for (int kc0 = 0; kc0 < kchunks; kc0 += CHAIN) {
        const int kc1 = kc0 + CHAIN < kchunks ? kc0 + CHAIN : kchunks;
        Acc128<BN> acc;
        int prev = -1;
        for (int kc = kc0; kc < kc1; ++kc) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_a + stage * STAGE, sb = sa + 4 * A_BOX;
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < KR / 16; ++ks) {      // 16 contraction rows (2048 B of an MN-major box) per MMA
            const uint32_t off = ks * 2048;
            const uint64_t ah0 = gmma_desc_mnmajor_sw128(sa + off, A_BOX);
            const uint64_t ah1 = gmma_desc_mnmajor_sw128(sa + A_BOX + off, A_BOX);
            const uint64_t al0 = gmma_desc_mnmajor_sw128(sa + 2 * A_BOX + off, A_BOX);
            const uint64_t al1 = gmma_desc_mnmajor_sw128(sa + 3 * A_BOX + off, A_BOX);
            uint64_t bh, bl;
            if (TB == 0) {
              bh = gmma_desc_kmajor_sw128(sb) + (uint64_t)(ks * 2);
              bl = gmma_desc_kmajor_sw128(sb + B_BYTES) + (uint64_t)(ks * 2);
            } else {
              bh = gmma_desc_mnmajor_sw128(sb + off, A_BOX);
              bl = gmma_desc_mnmajor_sw128(sb + B_BYTES + off, A_BOX);
            }
            acc.template mma<false, 1, TB>(al0, al1, bh, (kc > kc0 || ks > 0) ? 1u : 0u);
            acc.template mma<false, 1, TB>(ah0, ah1, bl, 1u);
            acc.template mma<false, 1, TB>(ah0, ah1, bh, 1u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        acc.fence_operands();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        // the finished chain: the first one stores, later ones load-add-store (each element has one owner thread)
#pragma unroll
        for (int ch = 0; ch < BN / 32; ++ch) {
          uint32_t raw[32];
          acc.rows32(ch, stg, raw);
          const int cn = g.cols - (c0 + ch * 32);         // output rows of this chunk that exist
          if (d < g.D && cn > 0) {
            float* o = g.out + (long long)(c0 + ch * 32) * g.D + d;
            if (kc0 == 0) {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (j < cn) o[(long long)j * g.D] = __uint_as_float(raw[j]);
            } else {
              // in groups of eight: 32 loads in flight next to the live accumulator would spill
#pragma unroll
              for (int j8 = 0; j8 < 32; j8 += 8) {
#pragma unroll
                for (int j = j8; j < j8 + 8; ++j)
                  if (j < cn) o[(long long)j * g.D] += __uint_as_float(raw[j]);
                asm volatile("" ::: "memory");
              }
            }
          }
        }
      }
    }
  }
}

template <int BN, int TB, int KR, int STAGES>
static int launch_pca_bwd_variant(const CUtensorMap* maps, const PcaBwdArgs& g, cudaStream_t s) {
  constexpr int smem = STAGES * PcaBwdShape<BN, TB, KR>::STAGE + ACC_STG_BYTES + 1024 + 256;
  static_assert(smem <= 232448, "shared-memory budget");
  auto kern = pca_bwd_tc_kernel<BN, TB, KR, STAGES>;
  static DeviceOnce attr_done;   // the attribute is per device
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_done.mark();
  }
  int per_sm = 1;
  IBL_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 160, smem));
  if (per_sm < 1) per_sm = 1;
  const int total = g.d_tiles * g.c_tiles;
  const int slots = per_sm * device_sm_count();
  kern<<<total < slots ? total : slots, 160, smem, s>>>(maps[0], maps[1], maps[2], maps[3], g);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// gv [N,D] = gy [N,P] . W [P,D].  W planes [P][D]; gy planes [N][Pp] (Pp = P rounded up to 8, zero columns).
int launch_pca_dgrad_tc(const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo, int P, int D, const __nv_bfloat16* g_hi,
                        const __nv_bfloat16* g_lo, int Pp, int N, float* gv, cudaStream_t s) {
  IBL_REQUIRE(D % 64 == 0 && Pp % 8 == 0 && Pp >= P, "tensor-core PCA dgrad needs D % 64 == 0");
  const int BN = N <= 32 ? 32 : (N <= 64 ? 64 : 128);
  CUtensorMap maps[4];
  {
    uint64_t dims[2] = {(uint64_t)D, (uint64_t)P}, str[1] = {(uint64_t)D * 2};
    uint32_t box[2] = {64, 64};
    IBL_RET(make_tmap(&maps[0], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, w_hi, dims, str, box));
    IBL_RET(make_tmap(&maps[1], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, w_lo, dims, str, box));
  }
  {
    uint64_t dims[2] = {(uint64_t)Pp, (uint64_t)N}, str[1] = {(uint64_t)Pp * 2};
    uint32_t box[2] = {64, (uint32_t)BN};
    IBL_RET(make_tmap(&maps[2], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, g_hi, dims, str, box));
    IBL_RET(make_tmap(&maps[3], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, g_lo, dims, str, box));
  }
  PcaBwdArgs g{};
  g.D = D; g.cols = N; g.K = P;
  g.d_tiles = cdiv(D, 128); g.c_tiles = cdiv(N, BN);
  g.out = gv;
  if (BN == 32) return launch_pca_bwd_variant<32, 0, 64, 4>(maps, g, s);
  if (BN == 64) return launch_pca_bwd_variant<64, 0, 64, 4>(maps, g, s);
  return launch_pca_bwd_variant<128, 0, 64, 3>(maps, g, s);
}

// gW [P,D] = gy^T [P,N] . v [N,D].  v planes [N][D]; gy planes [N][Pp].
int launch_pca_wgrad_tc(const __nv_bfloat16* v_hi, const __nv_bfloat16* v_lo, int N, int D, const __nv_bfloat16* g_hi,
                        const __nv_bfloat16* g_lo, int P, int Pp, float* gW, cudaStream_t s) {
  IBL_REQUIRE(D % 64 == 0 && Pp % 8 == 0 && Pp >= P, "tensor-core PCA wgrad needs D % 64 == 0");
  constexpr int KR = 16;
  CUtensorMap maps[4];
  uint32_t box[2] = {64, KR};
  {
    uint64_t dims[2] = {(uint64_t)D, (uint64_t)N}, str[1] = {(uint64_t)D * 2};
    IBL_RET(make_tmap(&maps[0], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, v_hi, dims, str, box));
    IBL_RET(make_tmap(&maps[1], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, v_lo, dims, str, box));
  }
  {
    uint64_t dims[2] = {(uint64_t)Pp, (uint64_t)N}, str[1] = {(uint64_t)Pp * 2};
    IBL_RET(make_tmap(&maps[2], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, g_hi, dims, str, box));
    IBL_RET(make_tmap(&maps[3], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, g_lo, dims, str, box));
  }
  PcaBwdArgs g{};
  g.D = D; g.cols = P; g.K = N;
  g.d_tiles = cdiv(D, 128); g.c_tiles = cdiv(P, 128);
  g.out = gW;
  return launch_pca_bwd_variant<128, 1, KR, 4>(maps, g, s);
}

// ---- CUDA-core helpers ------------------------------------------------------------------------------------------------
// gy [N,P] fp32 -> bf16 hi/lo planes [N][Pp], columns P..Pp-1 zero (TMA row strides are multiples of 16 bytes)
__global__ void pca_gy_planes_kernel(const float* __restrict__ gy, int N, int P, int Pp, __nv_bfloat16* __restrict__ hi,
                                     __nv_bfloat16* __restrict__ lo) {
  const long long total = (long long)N * Pp;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / Pp), p = (int)(i - (long long)n * Pp);
    const float v = p < P ? gy[(long long)n * P + p] : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}
int launch_pca_gy_planes(const float* gy, int N, int P, int Pp, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t s) {
  const long long total = (long long)N * Pp;
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  pca_gy_planes_kernel<<<(unsigned)(blocks > 0 ? blocks : 1), 256, 0, s>>>(gy, N, P, Pp, hi, lo);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// gb[p] = sum_n gy[n,p], rows in order
__global__ void pca_bias_grad_kernel(const float* __restrict__ gy, int N, int P, float* __restrict__ gb) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float acc = 0.f;
  for (int n = 0; n < N; ++n) acc += gy[(long long)n * P + p];
  gb[p] = acc;
}
int launch_pca_bias_grad(const float* gy, int N, int P, float* gb, cudaStream_t s) {
  pca_bias_grad_kernel<<<cdiv(P, 256), 256, 0, s>>>(gy, N, P, gb);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// fp32 math mode: C[r,d] = sum_k A[r*sr + k*sk] B[k,d] (B row-major [K,D]).  dgrad: r = n, k = p, A = gy (sr = P,
// sk = 1), B = W.  wgrad: r = p, k = n, A = gy (sr = 1, sk = P), B = v.  Thread = column d, 16 rows r per block row.
constexpr int TN_R = 16, TN_K = 64;
__global__ void __launch_bounds__(256)
pca_tn_simt_kernel(const float* __restrict__ A, long long sr, long long sk, int R, int K, const float* __restrict__ B,
                   int D, float* __restrict__ C) {
  __shared__ float a[TN_R][TN_K];
  const int d = blockIdx.x * 256 + threadIdx.x, r0 = blockIdx.y * TN_R;
  float acc[TN_R];
#pragma unroll
  for (int r = 0; r < TN_R; ++r) acc[r] = 0.f;
  for (int k0 = 0; k0 < K; k0 += TN_K) {
    for (int i = threadIdx.x; i < TN_R * TN_K; i += 256) {
      const int r = i / TN_K, k = i - r * TN_K;
      a[r][k] = (r0 + r < R && k0 + k < K) ? A[(r0 + r) * sr + (k0 + k) * sk] : 0.f;
    }
    __syncthreads();
    const int ke = K - k0 < TN_K ? K - k0 : TN_K;
    if (d < D) {
      for (int k = 0; k < ke; ++k) {
        const float b = __ldg(B + (long long)(k0 + k) * D + d);
#pragma unroll
        for (int r = 0; r < TN_R; ++r) acc[r] = fmaf(a[r][k], b, acc[r]);
      }
    }
    __syncthreads();
  }
  if (d < D) {
#pragma unroll
    for (int r = 0; r < TN_R; ++r)
      if (r0 + r < R) C[(long long)(r0 + r) * D + d] = acc[r];
  }
}
int launch_pca_tn_simt(const float* A, long long sr, long long sk, int R, int K, const float* B, int D, float* C,
                       cudaStream_t s) {
  dim3 grid((unsigned)cdiv(D, 256), (unsigned)cdiv(R, TN_R));
  pca_tn_simt_kernel<<<grid, 256, 0, s>>>(A, sr, sk, R, K, B, D, C);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

}  // namespace ibl
