// Image resize on the GPU, bit-exact with Pillow's 8-bit bilinear resample (SURVEY 8 f4: the reference's test transform
// starts with T.Resize((height, width)) on a PIL image, ibl/utils/data/__init__.py:37-42 -> PIL ImagingResample,
// antialiased two-pass convolution in fixed point).
//
// Pillow (src/libImaging/Resample.c): per output coordinate a window [xmin, xmin + xmax) of input samples and
// `ksize` coefficients, computed in double precision and rounded to integers with 22 fractional bits
// (PRECISION_BITS = 32 - 8 - 2); each pass accumulates  ss = 2^21 + sum pixel * coeff  in int32, shifts right by 22 and
// clamps to [0, 255]; horizontal pass first, its uint8 result feeds the vertical pass.  The coefficient tables are
// tiny and are built on the host exactly as Pillow does (openibl_b200/utils/data/gpu_resize.py); the passes below are
// integer work, one output pixel (3 channels) per thread.
#include "common.cuh"

namespace ibl {

constexpr int RS_PRECISION_BITS = 32 - 8 - 2;

__device__ __forceinline__ uint8_t rs_clip8(int v) {
  v >>= RS_PRECISION_BITS;                         // arithmetic shift, as the C code's lookup index
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// out[n, y, xo, c] = clip8(2^21 + sum_k in[n, y, xmin(xo) + k, c] * kk[xo][k])
__global__ void resize_h_u8_kernel(const uint8_t* __restrict__ in, int N, int H, int Win, int Wout,
                                   const int* __restrict__ bounds, const int* __restrict__ kk, int ksize,
                                   uint8_t* __restrict__ out) {
  const long long total = (long long)N * H * Wout;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xo = (int)(i % Wout);
    const long long row = i / Wout;                // n * H + y
    const int xmin = __ldg(bounds + 2 * xo), cnt = __ldg(bounds + 2 * xo + 1);
    const int* k = kk + (long long)xo * ksize;
    const uint8_t* p = in + (row * Win + xmin) * 3;
    int s0 = 1 << (RS_PRECISION_BITS - 1), s1 = s0, s2 = s0;
    for (int x = 0; x < cnt; ++x) {
      const int w = __ldg(k + x);
      s0 += (int)p[3 * x + 0] * w;
      s1 += (int)p[3 * x + 1] * w;
      s2 += (int)p[3 * x + 2] * w;
    }
    uint8_t* o = out + i * 3;
    o[0] = rs_clip8(s0); o[1] = rs_clip8(s1); o[2] = rs_clip8(s2);
  }
}

// out[n, yo, x, c] = clip8(2^21 + sum_k in[n, ymin(yo) + k, x, c] * kk[yo][k])
__global__ void resize_v_u8_kernel(const uint8_t* __restrict__ in, int N, int Hin, int Hout, int W,
                                   const int* __restrict__ bounds, const int* __restrict__ kk, int ksize,
                                   uint8_t* __restrict__ out) {
  const long long total = (long long)N * Hout * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const long long r = i / W;
    const int yo = (int)(r % Hout);
    const long long n = r / Hout;
    const int ymin = __ldg(bounds + 2 * yo), cnt = __ldg(bounds + 2 * yo + 1);
    const int* k = kk + (long long)yo * ksize;
    const uint8_t* p = in + ((n * Hin + ymin) * W + x) * 3;
    int s0 = 1 << (RS_PRECISION_BITS - 1), s1 = s0, s2 = s0;
    for (int y = 0; y < cnt; ++y) {
      const int w = __ldg(k + y);
      const uint8_t* q = p + (long long)y * W * 3;
      s0 += (int)q[0] * w;
      s1 += (int)q[1] * w;
      s2 += (int)q[2] * w;
    }
    uint8_t* o = out + i * 3;
    o[0] = rs_clip8(s0); o[1] = rs_clip8(s1); o[2] = rs_clip8(s2);
  }
}

// x [N,Hin,Win,3] u8 -> out [N,Hout,Wout,3]; tmp [N,Hin,Wout,3] (used when both passes run).  A pass whose sizes are
// equal is skipped (Pillow: need_horizontal / need_vertical); with both equal the image is copied.
int launch_resize_bilinear_u8(const uint8_t* x, int N, int Hin, int Win, int Hout, int Wout, const int* bounds_h,
                              const int* kk_h, int ksize_h, const int* bounds_v, const int* kk_v, int ksize_v,
                              uint8_t* tmp, uint8_t* out, cudaStream_t s, uint64_t* launches) {
  const bool need_h = Wout != Win, need_v = Hout != Hin;
  auto blocks = [](long long total) {
    long long b = (total + 255) / 256;
    return (unsigned)(b > 132 * 16 ? 132 * 16 : (b > 0 ? b : 1));
  };
  if (!need_h && !need_v) {
    IBL_CUDA_OK(cudaMemcpyAsync(out, x, (size_t)N * Hin * Win * 3, cudaMemcpyDeviceToDevice, s));
    return IBL_OK;
  }
  const uint8_t* src = x;
  if (need_h) {
    uint8_t* dst = need_v ? tmp : out;
    resize_h_u8_kernel<<<blocks((long long)N * Hin * Wout), 256, 0, s>>>(src, N, Hin, Win, Wout, bounds_h, kk_h, ksize_h, dst);
    src = dst;
    if (launches) ++*launches;
  }
  if (need_v) {
    resize_v_u8_kernel<<<blocks((long long)N * Hout * Wout), 256, 0, s>>>(src, N, Hin, Hout, Wout, bounds_v, kk_v, ksize_v, out);
    if (launches) ++*launches;
  }
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

}  // namespace ibl
