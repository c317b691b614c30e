// conv1_1 (Cin = 3, reference ibl/models/vgg.py slot 0) on the Hopper tensor cores (wgmma).
//
// K = 27 is too short for a TMA-fed implicit GEMM (a 3-channel NHWC row is 6 bytes), so the A
// operand is built in shared memory by four "im2col" warps straight from the NCHW fp32 input:
// one pixel per thread, its 3x3x3 window ordered k = tap*3 + c, split into bf16 hi/lo, zero-padded
// to K = 32 and written as one K-major 128-byte-swizzled row (the layout TMA would have produced).
// The 64x27 filter bank is laid out the same way once per CTA.  Two K=16 MMA steps x 3 (bf16x3)
// per 128-pixel tile; the epilogue is the usual accumulator -> bias -> ReLU -> hi/lo planes with
// 16-byte stores.  The kernel is bound by the 2.5 GB of NHWC output it writes per batch of 32.
//
// Warps: 0-3 consumer warpgroup (wgmma + epilogue), 4-7 operand builders.  A is double-buffered,
// persistent grid.
#include "common.cuh"
#include "tc_common.cuh"

namespace ibl {

using namespace tc;

struct Conv1Args {
  const float* x;       // [N,3,H,W]
  const float* w;       // OIHW [64,3,3,3]
  const float* bias;    // [64]
  __nv_bfloat16* y_hi;  // [N,H,W,64]
  __nv_bfloat16* y_lo;
  int N, H, W;
  int total_tiles;      // ceil(N*H*W / 128)
};

constexpr int C1_ABYTES = 128 * 128;   // one plane of one A stage: 128 rows x 128 B
constexpr int C1_OFF_A = 16384;                          // after the filters (hi 8 KiB | lo 8 KiB)
constexpr int C1_OFF_OUT = C1_OFF_A + 4 * C1_ABYTES;     // output staging: 4 warps x (hi 4 KiB | lo 4 KiB)
constexpr int C1_OFF_ACC = C1_OFF_OUT + 4 * 8192;        // accumulator transposition
constexpr int C1_OFF_BAR = C1_OFF_ACC + ACC_STG_BYTES;
constexpr int C1_SMEM = C1_OFF_BAR + 512 + 1024;

__global__ void __launch_bounds__(256, 1) conv1_1_tc_kernel(const Conv1Args a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* b_hi = smem;                       // [64 rows][128 B]
  uint8_t* b_lo = smem + 8192;
  uint8_t* a_buf = smem + C1_OFF_A;           // 2 stages x (hi 16 KiB | lo 16 KiB)
  uint8_t* stg = smem + C1_OFF_OUT;
  float* acc_stg = reinterpret_cast<float*>(smem + C1_OFF_ACC);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C1_OFF_BAR);
  uint64_t* a_full = bars;        // [2] count 4 (builder warps)
  uint64_t* a_empty = bars + 2;   // [2] count 4 (consumer warps)
  float* bias_s = reinterpret_cast<float*>(bars + 4);   // [64]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // zero both A stages once (the K >= 32 half of every row stays zero) and lay out the filters
  for (int i = threadIdx.x; i < (4 * C1_ABYTES) / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(a_buf)[i] = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < 64 * 8; i += blockDim.x) {   // (row n, chunk j): 8 k-values each
    const int n = i >> 3, j = i & 7;
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float v[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int k = j * 8 + e * 2 + u;          // k = tap*3 + c
        v[u] = 0.f;
        if (k < 27) v[u] = a.w[(n * 3 + (k % 3)) * 9 + (k / 3)];
      }
      const __nv_bfloat16 h0 = __float2bfloat16_rn(v[0]), h1 = __float2bfloat16_rn(v[1]);
      __nv_bfloat162 hh(h0, h1);
      __nv_bfloat162 ll = __floats2bfloat162_rn(v[0] - __bfloat162float(h0), v[1] - __bfloat162float(h1));
      hi[e] = *reinterpret_cast<uint32_t*>(&hh);
      lo[e] = *reinterpret_cast<uint32_t*>(&ll);
    }
    const int pos = n * 128 + ((j ^ (n & 7)) * 16);
    *reinterpret_cast<uint4*>(b_hi + pos) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(b_lo + pos) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
  if (threadIdx.x < 64) bias_s[threadIdx.x] = a.bias[threadIdx.x];
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) {
      mbar_init(&a_full[i], 4);
      mbar_init(&a_empty[i], 4);
    }
    fence_barrier_init();
  }
  fence_proxy_async();        // generic-proxy writes of B (and the zero fill) -> visible to the tensor core
  __syncthreads();
  const long long M = (long long)a.N * a.H * a.W;
  const long long HW = (long long)a.H * a.W;

  if (warp < 4) {
    // ---------------- consumer warpgroup: MMA + epilogue ----------------
    const uint64_t bh = gmma_desc_kmajor_sw128(smem_u32(b_hi)), bl = gmma_desc_kmajor_sw128(smem_u32(b_lo));
    int it = 0;
    for (int tile = blockIdx.x; tile < a.total_tiles; tile += gridDim.x, ++it) {
      const int st = it & 1;
      const uint32_t ph = (it >> 1) & 1;
      mbar_wait(&a_full[st], ph);
      const uint32_t sa = smem_u32(a_buf + st * 2 * C1_ABYTES);
      const uint64_t ah = gmma_desc_kmajor_sw128(sa), al = gmma_desc_kmajor_sw128(sa + C1_ABYTES);
      constexpr uint64_t kHalf = 64 * 128 / 16;   // pixel rows 64-127: +8 KiB
      Acc128<64> acc;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 2; ++k) {             // K = 32: two 16-wide steps (columns 32..63 are zero)
        const uint64_t ko = (uint64_t)(k * 2);
        acc.mma(al + ko, al + kHalf + ko, bh + ko, k > 0 ? 1u : 0u);
        acc.mma(ah + ko, ah + kHalf + ko, bl + ko, 1u);
        acc.mma(ah + ko, ah + kHalf + ko, bh + ko, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc.fence_operands();
      __syncwarp();
      if (lane == 0) mbar_arrive(&a_empty[st]);   // the builders may refill this stage
      // bias + ReLU + hi/lo split into this warp's staging rows (one 128-byte row per pixel and plane,
      // 16-byte chunks XOR-swizzled by the row index), then the warp writes its 32 pixels as eight fully
      // coalesced 512-byte stores per plane instead of 32 scattered 16-byte pieces per instruction.
      uint8_t* sth = stg + warp * 8192 + lane * 128;
      uint8_t* stl = sth + 4096;
#pragma unroll
      for (int ch = 0; ch < 2; ++ch) {
        uint32_t raw[32];
        acc.rows32(ch, acc_stg, raw);
        uint32_t hi[16], lo[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float x0 = fmaxf(__uint_as_float(raw[2 * j]) + bias_s[ch * 32 + 2 * j], 0.f);
          const float x1 = fmaxf(__uint_as_float(raw[2 * j + 1]) + bias_s[ch * 32 + 2 * j + 1], 0.f);
          const __nv_bfloat16 h0 = __float2bfloat16_rn(x0), h1 = __float2bfloat16_rn(x1);
          __nv_bfloat162 hh(h0, h1);
          __nv_bfloat162 ll = __floats2bfloat162_rn(x0 - __bfloat162float(h0), x1 - __bfloat162float(h1));
          hi[j] = *reinterpret_cast<uint32_t*>(&hh);
          lo[j] = *reinterpret_cast<uint32_t*>(&ll);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int pos = ((ch * 4 + j) ^ (lane & 7)) * 16;
          *reinterpret_cast<uint4*>(sth + pos) = make_uint4(hi[4 * j], hi[4 * j + 1], hi[4 * j + 2], hi[4 * j + 3]);
          *reinterpret_cast<uint4*>(stl + pos) = make_uint4(lo[4 * j], lo[4 * j + 1], lo[4 * j + 2], lo[4 * j + 3]);
        }
      }
      __syncwarp();
      {
        const uint8_t* wb = stg + warp * 8192;
        const long long p0 = (long long)tile * 128 + warp * 32;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int r = i * 4 + (lane >> 3), cchunk = lane & 7;
          const int pos = r * 128 + ((cchunk ^ (r & 7)) * 16);
          const uint4 vh = *reinterpret_cast<const uint4*>(wb + pos);
          const uint4 vl = *reinterpret_cast<const uint4*>(wb + 4096 + pos);
          if (p0 + r < M) {
            *reinterpret_cast<uint4*>(a.y_hi + (p0 + r) * 64 + cchunk * 8) = vh;
            *reinterpret_cast<uint4*>(a.y_lo + (p0 + r) * 64 + cchunk * 8) = vl;
          }
        }
      }
      __syncwarp();                               // the staging rows are rewritten by the next tile
    }
  } else {
    // ---------------- operand builders: one pixel (= one A row) per thread ----------------
    const int row = (warp - 4) * 32 + lane;
    int it = 0;
    for (int tile = blockIdx.x; tile < a.total_tiles; tile += gridDim.x, ++it) {
      const int st = it & 1;
      const uint32_t ph = (it >> 1) & 1;
      const long long pm = (long long)tile * 128 + row;
      float v[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) v[k] = 0.f;
      if (pm < M) {
        const long long n = pm / HW;
        const int rem = (int)(pm - n * HW);
        const int h = rem / a.W, w = rem - (rem / a.W) * a.W;
        const float* xb = a.x + n * 3 * HW;
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const int ih = h + tap / 3 - 1, iw = w + tap % 3 - 1;
          if (ih >= 0 && ih < a.H && iw >= 0 && iw < a.W) {
            const long long o = (long long)ih * a.W + iw;
#pragma unroll
            for (int c = 0; c < 3; ++c) v[tap * 3 + c] = __ldg(xb + c * HW + o);
          }
        }
      }
      mbar_wait(&a_empty[st], ph ^ 1);            // the MMAs that read this stage two tiles ago are done
      uint8_t* rh = a_buf + st * 2 * C1_ABYTES + row * 128;
      uint8_t* rl = rh + C1_ABYTES;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint32_t hi[4], lo[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float x0 = v[8 * j + 2 * e], x1 = v[8 * j + 2 * e + 1];
          const __nv_bfloat16 h0 = __float2bfloat16_rn(x0), h1 = __float2bfloat16_rn(x1);
          __nv_bfloat162 hh(h0, h1);
          __nv_bfloat162 ll = __floats2bfloat162_rn(x0 - __bfloat162float(h0), x1 - __bfloat162float(h1));
          hi[e] = *reinterpret_cast<uint32_t*>(&hh);
          lo[e] = *reinterpret_cast<uint32_t*>(&ll);
        }
        const int pos = (j ^ (row & 7)) * 16;
        *reinterpret_cast<uint4*>(rh + pos) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        *reinterpret_cast<uint4*>(rl + pos) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(&a_full[st]);
    }
  }
}

int launch_conv1_1_tc(const float* x_nchw, const float* w_oihw, const float* bias, int N, int H, int W,
                      __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, cudaStream_t s) {
  Conv1Args a{};
  a.x = x_nchw; a.w = w_oihw; a.bias = bias; a.y_hi = y_hi; a.y_lo = y_lo;
  a.N = N; a.H = H; a.W = W;
  const long long M = (long long)N * H * W;
  a.total_tiles = (int)((M + 127) / 128);
  static DeviceOnce attr_done;   // the attribute is per device
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(conv1_1_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C1_SMEM));
    attr_done.mark();
  }
  const int sms = device_sm_count();
  const int grid = a.total_tiles < sms ? a.total_tiles : sms;
  conv1_1_tc_kernel<<<grid, 256, C1_SMEM, s>>>(a);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

}  // namespace ibl
