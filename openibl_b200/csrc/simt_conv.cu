// CUDA-core (fp32) kernels of the backbone: the verification path of the 3x3 convolutions,
// conv1_1 (Cin=3, a K=27 contraction that does not tile onto a TMA-fed tensor-core GEMM), pooling and the
// layout changes at the boundary.  Reference: ibl/models/vgg.py:40-42,61-70.
#include "common.cuh"

namespace ibl {

// ------------------------------------------------------------------------------------------
// weight re-layout: OIHW fp32 -> [tap][Cin][Cout] fp32 (SIMT) and [tap][Cout][Cin] bf16 hi/lo (TC)
// ------------------------------------------------------------------------------------------
__global__ void repack_weights_kernel(const float* __restrict__ w, int cout, int cin,
                                      float* __restrict__ w_tck, __nv_bfloat16* __restrict__ w_hi,
                                      __nv_bfloat16* __restrict__ w_lo) {
  long long total = (long long)cout * cin * 9;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int tap = (int)(i % 9);
    long long r = i / 9;
    int ci = (int)(r % cin);
    int co = (int)(r / cin);
    float v = w[i];
    w_tck[((long long)tap * cin + ci) * cout + co] = v;
    if (w_hi) {
      __nv_bfloat16 h = __float2bfloat16_rn(v);
      __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
      long long o = ((long long)tap * cout + co) * cin + ci;
      w_hi[o] = h;
      w_lo[o] = l;
    }
  }
}

int launch_repack_weights(const float* w_oihw, int cout, int cin, ConvParams& p, cudaStream_t s) {
  long long total = (long long)cout * cin * 9;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  repack_weights_kernel<<<blocks, 256, 0, s>>>(w_oihw, cout, cin, p.w_tck, p.w_hi, p.w_lo);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ------------------------------------------------------------------------------------------
// generic 3x3 / stride 1 / pad 1 convolution, NHWC fp32, implicit GEMM on CUDA cores.
// M = N*H*W pixels, Ncol = Cout, K = 9*Cin.  Tile 128 x 64 x 16, 256 threads, 8x4 per thread.
// ------------------------------------------------------------------------------------------
constexpr int SC_BM = 128, SC_BN = 64, SC_BK = 16;

__global__ void __launch_bounds__(256)
conv3x3_simt_kernel(const float* __restrict__ x, const float* __restrict__ w,
                    const float* __restrict__ bias, float* __restrict__ y, int N, int H, int W,
                    int cin, int cout, int relu) {
  __shared__ __align__(16) float As[SC_BK][SC_BM];
  __shared__ __align__(16) float Bs[SC_BK][SC_BN];
  const int t = threadIdx.x;
  const int tn = t & 15, tm = t >> 4;
  const long long M = (long long)N * H * W;
  const long long m0 = (long long)blockIdx.x * SC_BM;
  const int n0 = blockIdx.y * SC_BN;

  const int lm = t & 127, kq0 = t >> 7;
  const long long pm = m0 + lm;
  const bool pvalid = pm < M;
  int ph = 0, pw = 0;
  long long pn = 0;
  if (pvalid) {
    pn = pm / ((long long)H * W);
    int rem = (int)(pm - pn * (long long)H * W);
    ph = rem / W;
    pw = rem - ph * W;
  }
  const int bk = t >> 4, bn = (t & 15) * 4;

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int tap = 0; tap < 9; ++tap) {
    const int ih = ph + tap / 3 - 1, iw = pw + tap % 3 - 1;
    const bool inb = pvalid && ih >= 0 && ih < H && iw >= 0 && iw < W;
    const float* xp = x + ((pn * H + ih) * (long long)W + iw) * cin;
    for (int c0 = 0; c0 < cin; c0 += SC_BK) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int kq = kq0 + 2 * j;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (inb) v = __ldg(reinterpret_cast<const float4*>(xp + c0 + kq * 4));
        As[kq * 4 + 0][lm] = v.x;
        As[kq * 4 + 1][lm] = v.y;
        As[kq * 4 + 2][lm] = v.z;
        As[kq * 4 + 3][lm] = v.w;
      }
      {
        float4 wv = __ldg(reinterpret_cast<const float4*>(
            w + ((long long)tap * cin + c0 + bk) * cout + n0 + bn));
        *reinterpret_cast<float4*>(&Bs[bk][bn]) = wv;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < SC_BK; ++k) {
        float4 a0 = *reinterpret_cast<const float4*>(&As[k][tm * 8]);
        float4 a1 = *reinterpret_cast<const float4*>(&As[k][tm * 8 + 4]);
        float4 b = *reinterpret_cast<const float4*>(&Bs[k][tn * 4]);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + n0 + tn * 4));
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long m = m0 + tm * 8 + i;
    if (m >= M) continue;
    float4 o;
    o.x = acc[i][0] + bv.x;
    o.y = acc[i][1] + bv.y;
    o.z = acc[i][2] + bv.z;
    o.w = acc[i][3] + bv.w;
    if (relu) {
      o.x = fmaxf(o.x, 0.f);
      o.y = fmaxf(o.y, 0.f);
      o.z = fmaxf(o.z, 0.f);
      o.w = fmaxf(o.w, 0.f);
    }
    *reinterpret_cast<float4*>(y + m * cout + n0 + tn * 4) = o;
  }
}

int launch_conv3x3_simt(const float* x, const ConvParams& p, int N, int H, int W, int cin,
                        int cout, bool relu, float* y, cudaStream_t s) {
  IBL_REQUIRE(cin % SC_BK == 0 && cout % SC_BN == 0, "conv3x3_simt needs Cin%16==0, Cout%64==0");
  long long M = (long long)N * H * W;
  dim3 grid((unsigned)((M + SC_BM - 1) / SC_BM), (unsigned)(cout / SC_BN));
  conv3x3_simt_kernel<<<grid, 256, 0, s>>>(x, p.w_tck, p.bias, y, N, H, W, cin, cout, relu ? 1 : 0);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ------------------------------------------------------------------------------------------
// conv1_1: NCHW fp32 [N,3,H,W] -> NHWC [N,H,W,64], + bias + ReLU (vgg.py slot 0).  K = 27 does not
// tile onto a TMA-fed tensor-core GEMM; this is the CUDA-core version: one pixel per thread, 64 accumulators in
// registers, the 27x64 weights broadcast from shared memory (LDS.128 feeds 4 FMAs).  Each thread
// writes its pixel's 64 fp32 channels as contiguous 16-byte stores, so every 128-byte line is fully
// written by one thread.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
conv1_1_kernel(const float* __restrict__ x, const float* __restrict__ w /*[27][64]*/,
               const float* __restrict__ bias, float* __restrict__ y, int N, int H, int W) {
  __shared__ __align__(16) float ws[27][64];
  __shared__ __align__(16) float bs[64];
  const int t = threadIdx.x;
  for (int i = t; i < 27 * 64; i += 128) ws[i / 64][i % 64] = w[i];   // w_tck: [tap][cin][cout]
  if (t < 64) bs[t] = bias[t];
  __syncthreads();
  const long long M = (long long)N * H * W;
  const long long pm = (long long)blockIdx.x * 128 + t;
  if (pm >= M) return;
  const long long pn = pm / ((long long)H * W);
  const int rem = (int)(pm - pn * (long long)H * W);
  const int ph = rem / W, pw = rem - (rem / W) * W;
  float acc[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = bs[j];
  float v[27];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int ih = ph + tap / 3 - 1, iw = pw + tap % 3 - 1;
    const bool inb = ih >= 0 && ih < H && iw >= 0 && iw < W;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      v[tap * 3 + c] = inb ? __ldg(x + ((pn * 3 + c) * H + ih) * (long long)W + iw) : 0.f;
  }
#pragma unroll
  for (int k = 0; k < 27; ++k) {
    const float4* wr = reinterpret_cast<const float4*>(ws[k]);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float4 wv = wr[j];
      acc[4 * j + 0] = fmaf(v[k], wv.x, acc[4 * j + 0]);
      acc[4 * j + 1] = fmaf(v[k], wv.y, acc[4 * j + 1]);
      acc[4 * j + 2] = fmaf(v[k], wv.z, acc[4 * j + 2]);
      acc[4 * j + 3] = fmaf(v[k], wv.w, acc[4 * j + 3]);
    }
  }
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = fmaxf(acc[j], 0.f);
  float4* o = reinterpret_cast<float4*>(y + pm * 64);
#pragma unroll
  for (int j = 0; j < 16; ++j) o[j] = make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
}

int launch_conv1_1(const float* x_nchw, const ConvParams& p, int N, int H, int W, float* y, cudaStream_t s) {
  long long M = (long long)N * H * W;
  unsigned blocks = (unsigned)((M + 127) / 128);
  conv1_1_kernel<<<blocks, 128, 0, s>>>(x_nchw, p.w_tck, p.bias, y, N, H, W);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ------------------------------------------------------------------------------------------
// MaxPool2d(2,2) floor mode, NHWC fp32
// ------------------------------------------------------------------------------------------
__global__ void maxpool2x2_kernel(const float4* __restrict__ x, float4* __restrict__ y, int N,
                                  int H, int W, int C4) {
  const int OH = H / 2, OW = W / 2;
  const long long total = (long long)N * OH * OW * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    long long r = i / C4;
    const int ow = (int)(r % OW);
    r /= OW;
    const int oh = (int)(r % OH);
    const long long n = r / OH;
    const float4* p = x + ((n * H + oh * 2) * (long long)W + ow * 2) * C4 + c;
    const float4 a = p[0], b = p[C4], cc = p[(long long)W * C4], d = p[(long long)W * C4 + C4];
    float4 o;
    o.x = fmaxf(fmaxf(a.x, b.x), fmaxf(cc.x, d.x));
    o.y = fmaxf(fmaxf(a.y, b.y), fmaxf(cc.y, d.y));
    o.z = fmaxf(fmaxf(a.z, b.z), fmaxf(cc.z, d.z));
    o.w = fmaxf(fmaxf(a.w, b.w), fmaxf(cc.w, d.w));
    y[i] = o;
  }
}

int launch_maxpool2x2(const float* x, int N, int H, int W, int C, float* y, cudaStream_t s) {
  IBL_REQUIRE(C % 4 == 0, "maxpool needs C%4==0");
  long long total = (long long)N * (H / 2) * (W / 2) * (C / 4);
  unsigned blocks = (unsigned)((total + 255) / 256);
  if (blocks > 132 * 32) blocks = 132 * 32;
  if (blocks == 0) blocks = 1;
  maxpool2x2_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const float4*>(x),
                                           reinterpret_cast<float4*>(y), N, H, W, C / 4);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ------------------------------------------------------------------------------------------
// [N,S,C] -> [N,C,S]   (the reference returns the feature map NCHW, vgg.py:70)
// ------------------------------------------------------------------------------------------
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int S,
                                    int C) {
  __shared__ float tile[32][33];
  const long long n = blockIdx.z;
  const int s0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int s = s0 + j, c = c0 + tx;
    if (s < S && c < C) tile[j][tx] = x[(n * S + s) * C + c];
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, s = s0 + tx;
    if (s < S && c < C) y[(n * C + c) * S + s] = tile[tx][j];
  }
}

int launch_nhwc_to_nchw(const float* x, int N, int S, int C, float* y, cudaStream_t s) {
  dim3 grid((unsigned)cdiv(S, 32), (unsigned)cdiv(C, 32), (unsigned)N);
  nhwc_to_nchw_kernel<<<grid, dim3(32, 8), 0, s>>>(x, y, S, C);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ToTensor + Normalize of the reference's test transform (ibl/utils/data/__init__.py:37-42, torchvision
// semantics): y[n,c,h,w] = ((x[n,h,w,c] / 255) - mean[c]) / std[c] with IEEE fp32 division and no contraction,
// so the result is bit-identical to the CPU transform.  uint8 HWC (decoder layout) -> fp32 NCHW.
// One thread per pixel: 3 byte loads (the warp covers 96 contiguous bytes), 3 coalesced plane stores.
__global__ void u8_hwc_to_nchw_norm_kernel(const uint8_t* __restrict__ x, float* __restrict__ y, long long hw,
                                           long long total, float m0, float m1, float m2, float s0, float s1,
                                           float s2) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / hw, p = i - n * hw;
    const uint8_t* px = x + i * 3;
    float* o = y + n * 3 * hw + p;
    o[0] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)px[0], 255.f), m0), s0);
    o[hw] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)px[1], 255.f), m1), s1);
    o[2 * hw] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)px[2], 255.f), m2), s2);
  }
}

int launch_u8_hwc_to_nchw_norm(const uint8_t* x, int N, int H, int W, const float* mean, const float* stdv, float* y,
                               cudaStream_t s) {
  const long long hw = (long long)H * W, total = hw * N;
  unsigned blocks = (unsigned)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (!blocks) blocks = 1;
  u8_hwc_to_nchw_norm_kernel<<<blocks, 256, 0, s>>>(x, y, hw, total, mean[0], mean[1], mean[2], stdv[0], stdv[1],
                                                    stdv[2]);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// AdaptiveMaxPool2d(1) over an NHWC map (vgg.py:67-68): [N,S,C] -> [N,C]
__global__ void global_maxpool_kernel(const float* __restrict__ x, float* __restrict__ y, int S,
                                      int C) {
  const long long n = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float m = -INFINITY;
  const float* p = x + n * S * (long long)C + c;
  for (int s = 0; s < S; ++s) m = fmaxf(m, p[(long long)s * C]);
  y[n * C + c] = m;
}

int launch_global_maxpool_nhwc(const float* x, int N, int S, int C, float* y, cudaStream_t s) {
  dim3 grid((unsigned)cdiv(C, 128), (unsigned)N);
  global_maxpool_kernel<<<grid, 128, 0, s>>>(x, y, S, C);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

__global__ void global_maxpool_planes_kernel(const __nv_bfloat16* __restrict__ hi,
                                             const __nv_bfloat16* __restrict__ lo, int S, int C,
                                             float* __restrict__ y) {
  const long long n = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float m = -INFINITY;
  const long long base = n * S * (long long)C + c;
  for (int s = 0; s < S; ++s) {
    const long long o = base + (long long)s * C;
    m = fmaxf(m, __bfloat162float(hi[o]) + __bfloat162float(lo[o]));
  }
  y[n * C + c] = m;
}
int launch_global_maxpool_planes(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int N, int S, int C, float* y,
                                 cudaStream_t s) {
  dim3 grid((unsigned)cdiv(C, 128), (unsigned)N);
  global_maxpool_planes_kernel<<<grid, 128, 0, s>>>(hi, lo, S, C, y);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// bf16 hi/lo planes <-> fp32
__global__ void planes_to_f32_kernel(const __nv_bfloat16* __restrict__ hi,
                                     const __nv_bfloat16* __restrict__ lo, size_t n,
                                     float* __restrict__ y) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x)
    y[i] = __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
}
__global__ void f32_to_planes_kernel(const float* __restrict__ x, size_t n,
                                     __nv_bfloat16* __restrict__ hi,
                                     __nv_bfloat16* __restrict__ lo) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}
int launch_planes_to_f32(const __nv_bfloat16* hi, const __nv_bfloat16* lo, size_t n, float* y,
                         cudaStream_t s) {
  unsigned blocks = (unsigned)((n + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (!blocks) blocks = 1;
  planes_to_f32_kernel<<<blocks, 256, 0, s>>>(hi, lo, n, y);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}
int launch_f32_to_planes(const float* x, size_t n, __nv_bfloat16* hi, __nv_bfloat16* lo,
                         cudaStream_t s) {
  unsigned blocks = (unsigned)((n + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (!blocks) blocks = 1;
  f32_to_planes_kernel<<<blocks, 256, 0, s>>>(x, n, hi, lo);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

}  // namespace ibl
