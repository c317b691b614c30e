// Hardware probe: does a K-major SWIZZLE_128B wgmma operand tolerate (a) a start address that is 128-byte
// but not 1024-byte aligned and (b) a stride between 8-row groups (SBO) that is not a multiple of 1024?
// That is what a convolution needs to read all nine taps out of ONE halo tile staged by a single TMA box
// ([rows of (TW+2) pixels][64 channels]): tap (kh,kw) starts (kh*(TW+2)+kw) rows into the tile and 8-pixel
// row groups are (TW+2) rows apart.
//
//   A_halo : [rows][64] bf16 dense, loaded by TMA with the 128B swizzle (row r at byte r*128, 16-byte chunk
//            j stored at chunk position j ^ (r & 7))
//   view   : row m of the 128-row operand = halo row  s0 + ((m % 64) / 8) * group_rows + (m / 64) * half_rows + (m % 8)
//            (half_rows = 8 * group_rows for a 16x8 patch, 8 for an 8x16 patch)
//   D[m,n] = sum_k view[m,k] * B[n,k]
// The caller compares D with the expected product for several (s0, group_rows, half_rows, base_offset mode).
// A second probe does the same for the 256-pixel kernel's register-A MMAs, whose B operand is the halo view.
#include "common.cuh"
#include "tc_common.cuh"

namespace ibl {

using namespace tc;

// K-major SW128 descriptor of the view starting at a_addr with 8-row groups sbo bytes apart; base_mode 1 sets the
// descriptor's base_offset field to the start row's swizzle phase
__device__ __forceinline__ uint64_t probe_desc(uint32_t a_addr, uint32_t sbo, int base_mode) {
  uint64_t d = 0;
  d |= (uint64_t)((a_addr >> 4) & 0x3fffu);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3fffu) << 32;
  if (base_mode == 1) d |= (uint64_t)((a_addr >> 7) & 7u) << 49;
  d |= (uint64_t)1 << 62;
  return d;
}

__global__ void __launch_bounds__(128, 1)
gmma_strided_probe_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                          int rows, int s0, int group_rows, int half_rows, int base_mode, float* __restrict__ D) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_sm = smem;                       // rows * 128 B (<= 32 KiB)
  uint8_t* b_sm = smem + 32768;               // 64 rows * 128 B
  float* stg = reinterpret_cast<float*>(smem + 32768 + 8192);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 32768 + 8192 + ACC_STG_BYTES);
  if (threadIdx.x == 0) {
    mbar_init(&bars[0], 1);
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bars[0], rows * 128 + 8192);
    tma_load_2d(a_sm, &tm_a, &bars[0], 0, 0);
    tma_load_2d(b_sm, &tm_b, &bars[0], 0, 0);
  }
  mbar_wait(&bars[0], 0);
  const uint32_t sbo = (uint32_t)group_rows * 128u;
  const uint32_t a0 = smem_u32(a_sm) + (uint32_t)s0 * 128u;
  const uint32_t a1 = a0 + (uint32_t)half_rows * 128u;   // rows 64-127 of the view
  const uint64_t da0 = probe_desc(a0, sbo, base_mode), da1 = probe_desc(a1, sbo, base_mode);
  const uint64_t db = gmma_desc_kmajor_sw128(smem_u32(b_sm));
  Acc128<64> acc;
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k)
    acc.mma(da0 + (uint64_t)(k * 2), da1 + (uint64_t)(k * 2), db + (uint64_t)(k * 2), k > 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  acc.fence_operands();
  float* o = D + (size_t)threadIdx.x * 64;
#pragma unroll
  for (int ch = 0; ch < 2; ++ch) {
    uint32_t r[32];
    acc.rows32(ch, stg, r);
#pragma unroll
    for (int j = 0; j < 32; ++j) o[ch * 32 + j] = __uint_as_float(r[j]);
  }
}

// A: [rows][64] bf16 bits, B: [64][64] bf16 bits (device), D: [128][64] fp32
int debug_gmma_strided(const void* A, int rows, const void* B, int s0, int group_rows, int half_rows, int base_mode,
                       float* D, cudaStream_t s) {
  IBL_REQUIRE(rows >= 8 && rows <= 256 && s0 >= 0 && group_rows >= 8 && half_rows >= 0 &&
                  s0 + half_rows + 7 * group_rows + 8 <= rows,
              "probe view does not fit the halo tile");
  CUtensorMap ma, mb;
  {
    uint64_t dims[2] = {64, (uint64_t)rows};
    uint64_t str[1] = {128};
    uint32_t box[2] = {64, (uint32_t)rows};
    IBL_RET(make_tmap(&ma, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, A, dims, str, box));
  }
  {
    uint64_t dims[2] = {64, 64};
    uint64_t str[1] = {128};
    uint32_t box[2] = {64, 64};
    IBL_RET(make_tmap(&mb, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, B, dims, str, box));
  }
  const int smem = 32768 + 8192 + ACC_STG_BYTES + 1024 + 64;
  static DeviceOnce attr_done;   // the attribute is per device
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(gmma_strided_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_done.mark();
  }
  gmma_strided_probe_kernel<<<1, 128, smem, s>>>(ma, mb, rows, s0, group_rows, half_rows, base_mode, D);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// Register-A probe (the 256-pixel conv kernel's operand roles): D[64 x n] = W . view(X)^T, one k16 step at a time for
// K = 64, with W's fragments read by ldsm_a_sw128 out of a TMA-staged SW128 [64][64] tile and the B operand an n64 or n128
// view of the halo tile X = [hrows][pitch][64] bf16: view row j is halo row s0 + (j / 8) * pitch + j % 8, 8-row groups
// pitch * 128 bytes apart (4352 B for the 8x32 patch's 34-pixel halo rows, 2304 B for the 16x16 patch's 18).
template <int N>
__global__ void __launch_bounds__(128, 1)
wgmma_rs_halo_probe_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x, int pitch,
                           int s0, uint32_t x_bytes, float* __restrict__ D) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* w_sm = smem;                       // 64 rows * 128 B
  uint8_t* x_sm = smem + 8192;                // hrows * pitch rows * 128 B (<= 44 KiB)
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 8192 + 45056);
  if (threadIdx.x == 0) {
    mbar_init(&bars[0], 1);
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bars[0], 8192 + x_bytes);
    tma_load_2d(w_sm, &tm_w, &bars[0], 0, 0);
    tma_load_3d(x_sm, &tm_x, &bars[0], 0, 0, 0);
  }
  mbar_wait(&bars[0], 0);
  const int t = threadIdx.x, lane = t & 31;
  const int row = 16 * (t >> 5) + (lane & 7) + 8 * ((lane >> 3) & 1);   // fragment row m reads W row m
  const uint64_t xd = ((uint64_t)1 << 16) | ((uint64_t)(((uint32_t)pitch * 128u) >> 4) << 32) | ((uint64_t)1 << 62) |
                      (uint64_t)(((smem_u32(x_sm) + (uint32_t)s0 * 128u) >> 4) & 0x3fffu);
  float d[N / 2];
  uint32_t f[4][4];
#pragma unroll
  for (int k = 0; k < 4; ++k) ldsm_a_sw128(f[k], smem_u32(w_sm), row, k);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) WgmmaRS<N>::mma(d, f[k], xd + (uint64_t)(k * 2), k > 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < N / 2; ++i) asm volatile("" : "+f"(d[i])::"memory");
  // accumulator layout: [4i + e] = (row 16 w + lane / 4 + 8 (e >> 1), column 8 i + 2 (lane % 4) + (e & 1))
  const int r0 = 16 * (t >> 5) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < N / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) D[(size_t)(r0 + 8 * (e >> 1)) * N + 8 * i + c0 + (e & 1)] = d[4 * i + e];
}

// W: [64][64] bf16 bits, X: [hrows][pitch][64] bf16 bits (device), D: [64][n] fp32
int debug_wgmma_rs_halo(const void* W, const void* X, int pitch, int hrows, int n, int s0, float* D, cudaStream_t s) {
  IBL_REQUIRE(n == 64 || n == 128, "probe view: n is 64 or 128");
  IBL_REQUIRE(pitch >= 8 && pitch <= 256 && hrows >= 1 && hrows <= 256 && pitch * hrows <= 352 && s0 >= 0 &&
                  s0 + (n / 8 - 1) * pitch + 8 <= pitch * hrows,
              "probe view does not fit the halo tile");
  CUtensorMap mw, mx;
  {
    uint64_t dims[2] = {64, 64};
    uint64_t str[1] = {128};
    uint32_t box[2] = {64, 64};
    IBL_RET(make_tmap(&mw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, W, dims, str, box));
  }
  {
    uint64_t dims[3] = {64, (uint64_t)pitch, (uint64_t)hrows};
    uint64_t str[2] = {128, (uint64_t)pitch * 128};
    uint32_t box[3] = {64, (uint32_t)pitch, (uint32_t)hrows};
    IBL_RET(make_tmap(&mx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, X, dims, str, box));
  }
  const int smem = 8192 + 45056 + 1024 + 64;
  const uint32_t x_bytes = (uint32_t)pitch * (uint32_t)hrows * 128u;
  if (n == 64) {
    static DeviceOnce attr_done;
    if (!attr_done.done()) {
      IBL_CUDA_OK(cudaFuncSetAttribute(wgmma_rs_halo_probe_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      attr_done.mark();
    }
    wgmma_rs_halo_probe_kernel<64><<<1, 128, smem, s>>>(mw, mx, pitch, s0, x_bytes, D);
  } else {
    static DeviceOnce attr_done;
    if (!attr_done.done()) {
      IBL_CUDA_OK(cudaFuncSetAttribute(wgmma_rs_halo_probe_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      attr_done.mark();
    }
    wgmma_rs_halo_probe_kernel<128><<<1, 128, smem, s>>>(mw, mx, pitch, s0, x_bytes, D);
  }
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

}  // namespace ibl
