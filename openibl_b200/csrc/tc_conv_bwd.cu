// Backward of the 3x3 / stride 1 / pad 1 convolutions of the VGG16 trunk (SURVEY 8 row f1: config 5 trains
// conv5_1..conv5_3 under the SFRS loss; reference: autograd through ibl/models/vgg.py:61-62, cuDNN dgrad/wgrad).
//
//   dgrad   dX[n,h,w,ci] = sum_{tap,co} dY[n,h-(kh-1),w-(kw-1),co] W[co,ci,kh,kw]
//           = the SAME tensor-core implicit-GEMM forward kernel (tc_conv.cu) applied to dY with the filter bank
//             rotated by 180 degrees and its channel roles swapped (repack_weights_dgrad_kernel).
//   wgrad   dW[co,ci,kh,kw] = sum_{n,h,w} dY[n,h,w,co] X[n,h+kh-1,w+kw-1,ci]
//           = per tap a GEMM whose reduction index is the PIXEL: both operands are "MN-major" in shared memory
//             (rows = pixels, 64 contiguous channels per 128-byte row), exactly what a TMA box of the NHWC
//             hi/lo planes delivers -- the layout the second NetVLAD contraction already uses (tc_netvlad.cu).
//             conv_wgrad_tc_kernel: one CTA per (tap, 128 output channels, 128 input channels, pixel split);
//             64-pixel K steps (boxes of 16 x 4 pixels; the X box is shifted by the tap, TMA zero-fills the
//             padding), bf16x3, one 128 x 128 fp32 wgmma accumulator restarted every WG_CHAIN_BOXES boxes and
//             added into the split's partial sum, partial sums per split reduced by wgrad_reduce_kernel into the
//             OIHW gradient.
//   db, ReLU mask, 2x2 max-pool backward: small CUDA-core kernels.
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace ibl {

using namespace tc;

// ---- filter bank for dgrad: planes [tap'][Cin][Cout] with tap' = 8 - tap (the forward kernel's [tap][N][K] layout with
// N = Cin, K = Cout), from the engine's fp32 copy w_tck [tap][Cin][Cout] ------------------------------------------
__global__ void repack_weights_dgrad_kernel(const float* __restrict__ w_tck, long long per_tap,
                                            __nv_bfloat16* __restrict__ w_hi, __nv_bfloat16* __restrict__ w_lo) {
  const long long total = per_tap * 9;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int tap = (int)(i / per_tap);
    const long long r = i - (long long)tap * per_tap;
    const float v = w_tck[i];
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    const long long o = (long long)(8 - tap) * per_tap + r;
    w_hi[o] = h;
    w_lo[o] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}
int launch_repack_weights_dgrad(const float* w_tck, int cout, int cin, __nv_bfloat16* w_hi, __nv_bfloat16* w_lo,
                                cudaStream_t s) {
  const long long per_tap = (long long)cout * cin;
  int blocks = (int)((per_tap * 9 + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  repack_weights_dgrad_kernel<<<blocks, 256, 0, s>>>(w_tck, per_tap, w_hi, w_lo);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ---- ReLU backward fused with the hi/lo split of dY (the operand format of both dgrad and wgrad) ---------------
// g_pre = g * (y > 0) if relu (y = post-ReLU output), planes + optional fp32 copy
__global__ void relu_mask_planes_kernel(const float* __restrict__ g, const float* __restrict__ y, size_t n, int relu,
                                        __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = g[i];
    if (relu && !(y[i] > 0.f)) v = 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}
int launch_relu_mask_planes(const float* g, const float* y, size_t n, bool relu, __nv_bfloat16* hi, __nv_bfloat16* lo,
                            cudaStream_t s) {
  unsigned blocks = (unsigned)((n + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (!blocks) blocks = 1;
  relu_mask_planes_kernel<<<blocks, 256, 0, s>>>(g, y, n, relu ? 1 : 0, hi, lo);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ---- bias gradient: db[co] = sum over pixels of dY (from the planes, i.e. after the ReLU mask) ----------------
__global__ void __launch_bounds__(256)
bias_grad_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, long long P, int C,
                 float* __restrict__ part /*[gridDim.x][C]*/) {
  // block b sums pixels b, b+grid, ...; thread t owns channels t, t+256, ...
  for (int c = threadIdx.x; c < C; c += 256) {
    float acc = 0.f;
    for (long long p = blockIdx.x; p < P; p += gridDim.x)
      acc += __bfloat162float(hi[p * C + c]) + __bfloat162float(lo[p * C + c]);
    part[(long long)blockIdx.x * C + c] = acc;
  }
}
__global__ void bias_grad_reduce_kernel(const float* __restrict__ part, int parts, int C, float* __restrict__ db) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float acc = 0.f;
  for (int p = 0; p < parts; ++p) acc += part[(long long)p * C + c];
  db[c] = acc;
}

// ---- 2x2 max-pool backward, NHWC fp32: the gradient goes to the FIRST maximum in row-major window order -----------
__global__ void maxpool2x2_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gy, int N, int H, int W,
                                      int C, float* __restrict__ gx) {
  const int OH = H / 2, OW = W / 2;
  const long long total = (long long)N * H * W * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int w = (int)(r % W);
    r /= W;
    const int h = (int)(r % H);
    const long long n = r / H;
    const int oh = h >> 1, ow = w >> 1;
    float out = 0.f;
    if (oh < OH && ow < OW) {
      const long long base = ((n * H + oh * 2) * (long long)W + ow * 2) * C + c;
      const float v00 = x[base], v01 = x[base + C], v10 = x[base + (long long)W * C], v11 = x[base + (long long)W * C + C];
      int arg = 0;
      float best = v00;
      if (v01 > best) { best = v01; arg = 1; }
      if (v10 > best) { best = v10; arg = 2; }
      if (v11 > best) { best = v11; arg = 3; }
      if (arg == ((h & 1) * 2 + (w & 1))) out = gy[((n * OH + oh) * (long long)OW + ow) * C + c];
    }
    gx[i] = out;
  }
}
int launch_maxpool2x2_bwd(const float* x, const float* gy, int N, int H, int W, int C, float* gx, cudaStream_t s) {
  const long long total = (long long)N * H * W * C;
  unsigned blocks = (unsigned)((total + 255) / 256);
  if (blocks > 132 * 32) blocks = 132 * 32;
  if (!blocks) blocks = 1;
  maxpool2x2_bwd_kernel<<<blocks, 256, 0, s>>>(x, gy, N, H, W, C, gx);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ---- wgrad on the tensor cores ----------------------------------------------------------------------------------------
struct WgradArgs {
  int N, H, W, cin, cout;
  int tiles_w, tiles_h;        // 16 x 4-pixel boxes per image
  int m_tiles, n_tiles;        // ceil(cout / 128), ceil(cin / 128)
  int splits;                  // pixel-range splits
  long long boxes;             // N * tiles_h * tiles_w
  float* part;                 // [splits][9][cout][cin]
};

constexpr int WG_BOX = 8192;                    // [64 px][64 ch] bf16
constexpr int WG_STAGE = 8 * WG_BOX;            // dY hi c0,c1 | dY lo c0,c1 | X hi c0,c1 | X lo c0,c1 = 64 KiB
constexpr int WG_STAGES = 3;
// The wgmma fp32 accumulator loses a little toward zero on every accumulation: a sum of positive products over one
// chain comes out smaller by ~3e-8 per MMA (measured on H100: 1e-3 after the 23,040 MMAs of a 1,920-box chain).  The
// consumer therefore restarts its chain every WG_CHAIN_BOXES boxes (96 MMAs) and adds the finished chain into its own
// [128 x 128] slice of the split's partial with ordinary fp32 adds, in a fixed order.
constexpr int WG_CHAIN_BOXES = 8;

__global__ void __launch_bounds__(160, 1)
conv_wgrad_tc_kernel(const __grid_constant__ CUtensorMap tm_ghi, const __grid_constant__ CUtensorMap tm_glo,
                     const __grid_constant__ CUtensorMap tm_xhi, const __grid_constant__ CUtensorMap tm_xlo,
                     const WgradArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* stg = reinterpret_cast<float*>(smem + WG_STAGES * WG_STAGE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + WG_STAGES * WG_STAGE + ACC_STG_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + WG_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // item = ((split * 9 + tap) * m_tiles + mt) * n_tiles + nt
  int item = blockIdx.x;
  const int nt = item % a.n_tiles; item /= a.n_tiles;
  const int mt = item % a.m_tiles; item /= a.m_tiles;
  const int tap = item % 9;
  const int split = item / 9;
  const int kh = tap / 3, kw = tap % 3;
  const long long per = (a.boxes + a.splits - 1) / a.splits;
  const long long b0 = (long long)split * per, b1 = (b0 + per < a.boxes) ? b0 + per : a.boxes;

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tm_ghi); tma_prefetch_desc(&tm_glo); tma_prefetch_desc(&tm_xhi); tma_prefetch_desc(&tm_xlo);
    for (int i = 0; i < WG_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  if (warp == 4) {
    // producer: the whole warp walks the loop in convergent code and ONE ELECTED lane (elect.sync) issues a stage's
    // TMA instructions, with ring position and addresses made warp-uniform
    const uint32_t smem_a = warp_uniform(smem_u32(smem));
    const uint32_t full_a = smem_a + WG_STAGES * WG_STAGE + ACC_STG_BYTES, empty_a = full_a + 8 * WG_STAGES;
    int stage = 0; uint32_t phase = 0;
    const int per_img = a.tiles_h * a.tiles_w;
    const int co0 = mt * 128, ci0 = nt * 128;
    for (long long b = b0; b < b1; ++b) {
      const int n = (int)(b / per_img);
      const int r = (int)(b - (long long)n * per_img);
      const int nu = (int)warp_uniform((uint32_t)n);
      const int h0 = (int)warp_uniform((uint32_t)((r / a.tiles_w) * 4)), w0 = (int)warp_uniform((uint32_t)((r % a.tiles_w) * 16));
      const uint32_t sg = warp_uniform((uint32_t)stage);
      mbar_wait_warp_a(empty_a + 8 * sg, phase ^ 1);
      const uint32_t st = smem_a + sg * WG_STAGE, fb = full_a + 8 * sg;
      if (elect_one()) {
        mbar_arrive_expect_tx_a(fb, WG_STAGE);
        tma_load_4d_a(st + 0 * WG_BOX, &tm_ghi, fb, co0, w0, h0, nu);
        tma_load_4d_a(st + 1 * WG_BOX, &tm_ghi, fb, co0 + 64, w0, h0, nu);
        tma_load_4d_a(st + 2 * WG_BOX, &tm_glo, fb, co0, w0, h0, nu);
        tma_load_4d_a(st + 3 * WG_BOX, &tm_glo, fb, co0 + 64, w0, h0, nu);
        tma_load_4d_a(st + 4 * WG_BOX, &tm_xhi, fb, ci0, w0 + kw - 1, h0 + kh - 1, nu);
        tma_load_4d_a(st + 5 * WG_BOX, &tm_xhi, fb, ci0 + 64, w0 + kw - 1, h0 + kh - 1, nu);
        tma_load_4d_a(st + 6 * WG_BOX, &tm_xlo, fb, ci0, w0 + kw - 1, h0 + kh - 1, nu);
        tma_load_4d_a(st + 7 * WG_BOX, &tm_xlo, fb, ci0 + 64, w0 + kw - 1, h0 + kh - 1, nu);
      }
      __syncwarp();
      if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
    }
  } else {
    // consumer warpgroup: D[co][ci] over the pixel range, both operands MN-major; then thread = output channel row
    const int co = mt * 128 + threadIdx.x;
    float* po = a.part + (((long long)split * 9 + tap) * a.cout + co) * a.cin + nt * 128;
    if (b1 > b0) {
      const uint32_t smem_a = smem_u32(smem);
      Acc128<128> acc;
      int stage = 0; uint32_t phase = 0;
      int prev = -1;
      for (long long c0 = b0; c0 < b1; c0 += WG_CHAIN_BOXES) {
        const long long c1 = (c0 + WG_CHAIN_BOXES < b1) ? c0 + WG_CHAIN_BOXES : b1;
        for (long long b = c0; b < c1; ++b) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_a + stage * WG_STAGE;
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {          // 16 pixel rows (2048 B) per MMA
            const uint32_t off = ks * 2048;
            // A = dY: output channels 0-63 / 64-127 of the tile are the two 64-channel boxes (one MN atom each)
            const uint64_t gh0 = gmma_desc_mnmajor_sw128(sa + off, WG_BOX);
            const uint64_t gh1 = gmma_desc_mnmajor_sw128(sa + WG_BOX + off, WG_BOX);
            const uint64_t gl0 = gmma_desc_mnmajor_sw128(sa + 2 * WG_BOX + off, WG_BOX);
            const uint64_t gl1 = gmma_desc_mnmajor_sw128(sa + 3 * WG_BOX + off, WG_BOX);
            // B = X: 128 input channels = two MN atoms WG_BOX apart
            const uint64_t xh = gmma_desc_mnmajor_sw128(sa + 4 * WG_BOX + off, WG_BOX);
            const uint64_t xl = gmma_desc_mnmajor_sw128(sa + 6 * WG_BOX + off, WG_BOX);
            acc.mma<false, 1, 1>(gl0, gl1, xh, (b == c0 && ks == 0) ? 0u : 1u);
            acc.mma<false, 1, 1>(gh0, gh1, xl, 1u);
            acc.mma<false, 1, 1>(gh0, gh1, xh, 1u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
          prev = stage;
          if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        acc.fence_operands();
        // the finished chain -> this thread's row of the slice: the first chain stores, later ones load-add-store
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
          uint32_t r[32];
          acc.rows32(ch, stg, r);
          if (co < a.cout) {
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const int ci = nt * 128 + ch * 32 + j;
              if (ci < a.cin) po[ch * 32 + j] = (c0 == b0 ? 0.f : po[ch * 32 + j]) + __uint_as_float(r[j]);
            }
          }
        }
      }
    } else if (co < a.cout) {
      for (int j = 0; j < 128; ++j)
        if (nt * 128 + j < a.cin) po[j] = 0.f;
    }
  }
}

// dW[co][ci][kh][kw] = sum_s part[s][tap][co][ci]
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int splits, int cout, int cin,
                                    float* __restrict__ dw_oihw) {
  const long long total = (long long)cout * cin * 9;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    // i indexes [tap][co][ci] so that reads are coalesced
    const int ci = (int)(i % cin);
    long long r = i / cin;
    const int co = (int)(r % cout);
    const int tap = (int)(r / cout);
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += part[(((long long)s * 9 + tap) * cout + co) * cin + ci];
    dw_oihw[((long long)co * cin + ci) * 9 + tap] = acc;
  }
}

int wgrad_tc_splits(int N, int H, int W, int cin, int cout) {
  const long long items = 9ll * cdiv(cout, 128) * cdiv(cin, 128);
  const long long boxes = (long long)N * cdiv(H, 4) * cdiv(W, 16);
  long long s = (2ll * device_sm_count() + items - 1) / items;      // about two waves of CTAs
  if (s < 1) s = 1;
  if (s > boxes) s = boxes > 0 ? boxes : 1;
  if (s > 64) s = 64;
  return (int)s;
}

// dY planes [N,H,W,cout], X planes [N,H,W,cin] (NHWC bf16 hi/lo) -> dw_oihw [cout,cin,3,3], db [cout] (nullable)
// part: [splits*9*cout*cin] floats; bpart: [256*cout] floats
int launch_conv_wgrad_tc(const __nv_bfloat16* g_hi, const __nv_bfloat16* g_lo, const __nv_bfloat16* x_hi,
                         const __nv_bfloat16* x_lo, int N, int H, int W, int cin, int cout, float* part, int splits,
                         float* bpart, float* dw_oihw, float* db, cudaStream_t s) {
  IBL_REQUIRE(cin % 64 == 0 && cout % 64 == 0, "tensor-core wgrad needs Cin%64==0 and Cout%64==0");
  CUtensorMap m_ghi, m_glo, m_xhi, m_xlo;
  {
    uint64_t dims[4] = {(uint64_t)cout, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t str[3] = {(uint64_t)cout * 2, (uint64_t)W * cout * 2, (uint64_t)H * W * cout * 2};
    uint32_t box[4] = {64, 16, 4, 1};
    IBL_RET(make_tmap(&m_ghi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, g_hi, dims, str, box));
    IBL_RET(make_tmap(&m_glo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, g_lo, dims, str, box));
  }
  {
    uint64_t dims[4] = {(uint64_t)cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t str[3] = {(uint64_t)cin * 2, (uint64_t)W * cin * 2, (uint64_t)H * W * cin * 2};
    uint32_t box[4] = {64, 16, 4, 1};
    IBL_RET(make_tmap(&m_xhi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x_hi, dims, str, box));
    IBL_RET(make_tmap(&m_xlo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x_lo, dims, str, box));
  }
  WgradArgs a{};
  a.N = N; a.H = H; a.W = W; a.cin = cin; a.cout = cout;
  a.tiles_w = cdiv(W, 16); a.tiles_h = cdiv(H, 4);
  a.m_tiles = cdiv(cout, 128); a.n_tiles = cdiv(cin, 128);
  a.splits = splits;
  a.boxes = (long long)N * a.tiles_h * a.tiles_w;
  a.part = part;
  const int smem = WG_STAGES * WG_STAGE + ACC_STG_BYTES + 1024 + 128;
  static DeviceOnce attr_done;
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(conv_wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_done.mark();
  }
  const int grid = splits * 9 * a.m_tiles * a.n_tiles;
  conv_wgrad_tc_kernel<<<grid, 160, smem, s>>>(m_ghi, m_glo, m_xhi, m_xlo, a);
  IBL_CUDA_OK(cudaGetLastError());
  const long long total = (long long)cout * cin * 9;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  wgrad_reduce_kernel<<<blocks, 256, 0, s>>>(part, splits, cout, cin, dw_oihw);
  IBL_CUDA_OK(cudaGetLastError());
  if (db) {
    const long long P = (long long)N * H * W;
    const int parts = P < 256 ? (int)P : 256;
    bias_grad_kernel<<<parts, 256, 0, s>>>(g_hi, g_lo, P, cout, bpart);
    bias_grad_reduce_kernel<<<cdiv(cout, 128), 128, 0, s>>>(bpart, parts, cout, db);
    IBL_CUDA_OK(cudaGetLastError());
  }
  return IBL_OK;
}

// ---- conv1_1 (Cin = 3) weight gradient: 64 x 27 outputs, reduction over every pixel; CUDA cores ---------------------
// block b sums pixels b*chunk .. ; thread t = (co = t & 63, quarter = t >> 6) strides the chunk by 4
__global__ void __launch_bounds__(256)
conv1_1_wgrad_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ g_hi,
                     const __nv_bfloat16* __restrict__ g_lo, int N, int H, int W, float* __restrict__ part /*[grid][64][28]*/) {
  __shared__ float red[4][64][28];
  const int co = threadIdx.x & 63, qd = threadIdx.x >> 6;
  const long long HW = (long long)H * W, P = (long long)N * HW;
  const long long chunk = (P + gridDim.x - 1) / gridDim.x;
  const long long p0 = (long long)blockIdx.x * chunk, p1 = (p0 + chunk < P) ? p0 + chunk : P;
  float acc[28];
#pragma unroll
  for (int k = 0; k < 28; ++k) acc[k] = 0.f;
  for (long long p = p0 + qd; p < p1; p += 4) {
    const float gv = __bfloat162float(g_hi[p * 64 + co]) + __bfloat162float(g_lo[p * 64 + co]);
    acc[27] += gv;                                   // bias gradient
    const long long n = p / HW;
    const int rem = (int)(p - n * HW);
    const int h = rem / W, w = rem - (rem / W) * W;
    const float* xb = x + n * 3 * HW;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int ih = h + tap / 3 - 1, iw = w + tap % 3 - 1;
      if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
        const long long o = (long long)ih * W + iw;
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c * 9 + tap] = fmaf(gv, __ldg(xb + c * HW + o), acc[c * 9 + tap]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 28; ++k) red[qd][co][k] = acc[k];
  __syncthreads();
  for (int i = threadIdx.x; i < 64 * 28; i += 256) {
    const int c2 = i / 28, k = i - c2 * 28;
    part[(long long)blockIdx.x * 64 * 28 + i] = (red[0][c2][k] + red[1][c2][k]) + (red[2][c2][k] + red[3][c2][k]);
  }
}
__global__ void conv1_1_wgrad_reduce_kernel(const float* __restrict__ part, int parts, float* __restrict__ dw,
                                            float* __restrict__ db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;   // (co, k) with k = c*9 + tap, or k = 27 for the bias
  if (i >= 64 * 28) return;
  float acc = 0.f;
  for (int p = 0; p < parts; ++p) acc += part[(long long)p * 64 * 28 + i];
  const int co = i / 28, k = i - co * 28;
  if (k == 27) db[co] = acc;
  else dw[co * 27 + k] = acc;                            // OIHW [64][3][3][3]: (c*9 + tap) is the row-major offset
}
int launch_conv1_1_wgrad(const float* x_nchw, const __nv_bfloat16* g_hi, const __nv_bfloat16* g_lo, int N, int H, int W,
                         float* part, float* dw_oihw, float* db, cudaStream_t s) {
  const long long P = (long long)N * H * W;
  const int parts = P < 1024 ? (int)P : 1024;
  conv1_1_wgrad_kernel<<<parts, 256, 0, s>>>(x_nchw, g_hi, g_lo, N, H, W, part);
  conv1_1_wgrad_reduce_kernel<<<cdiv(64 * 28, 128), 128, 0, s>>>(part, parts, dw_oihw, db);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

}  // namespace ibl
