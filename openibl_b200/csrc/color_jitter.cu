// T.ColorJitter on decoded uint8 HWC RGB images, bit-identical to torchvision's PIL path (the training transform's
// first step, ibl/utils/data/__init__.py:29-35).  ColorJitter.forward draws a random order of brightness, contrast,
// saturation and hue and applies each through Pillow:
//   brightness  ImageEnhance.Brightness = Image.blend(black, img, f)
//   contrast    ImageEnhance.Contrast   = Image.blend(mean of convert('L'), img, f)
//   saturation  ImageEnhance.Color      = Image.blend(convert('L').convert('RGB'), img, f)
//   hue         torchvision adjust_hue  = convert('HSV'), H += uint8(int32(f * 255)), convert('RGB')
// The per-pixel code restates Pillow's C (Blend.c ImagingBlend, Convert.c L24 / rgb2hsv_row / hsv2rgb) with its exact
// mix of float and double: every operation is an explicit round-to-nearest intrinsic, so no FMA contraction or fast-math
// flag can change a result.
//
// Contrast is the only step that needs the whole image (the mean of L at that point of the chain), and every chain has
// exactly one contrast step, so a batch takes two launches whatever its image sizes:
//   1. color_jitter_pre_kernel   the steps before contrast, per pixel; each block adds its pixels' L to the image's
//                                64-bit sum (integer atomics: exact in any order)
//   2. color_jitter_post_kernel  mean = int(sum / count + 0.5) in double, then contrast and the remaining steps
// Blocks are dealt to images by a host-built table of first blocks, so one launch covers mixed sizes without idle blocks.
#include <math.h>
#include <string.h>

#include <new>
#include <vector>

#include "common.cuh"

namespace ibl {

namespace {

constexpr int kThreads = 256;
constexpr int kPixPerThread = 4;
constexpr int kPixPerBlock = kThreads * kPixPerThread;

enum : int { kBrightness = 0, kContrast = 1, kSaturation = 2, kHue = 3 };

struct JitterImg {
  unsigned long long off;     // byte offset of the image in the caller's buffer
  unsigned long long npix;
  unsigned block0;            // first block of the image in either launch
  int n_pre, n_post;          // steps before / after the contrast step
  unsigned pre, post;         // their op codes, 4 bits each, first step in the low bits
  int contrast;               // 1: the chain has a contrast step (its factor is not None)
  float bright, contr, sat;
  int hue_shift;              // uint8(int32(hue * 255))
};

__device__ __forceinline__ int clip8(int v) { return v <= 0 ? 0 : (v < 256 ? v : 255); }

// Image.blend(deg, img, a): out = (UINT8)(deg + a * (img - deg)) in float; clipped when a is outside [0, 1]
__device__ __forceinline__ int blend1(int deg, int img, float a) {
  const float t = __fadd_rn((float)deg, __fmul_rn(a, (float)(img - deg)));
  if (a >= 0.f && a <= 1.f) return (int)t;
  if (t <= 0.f) return 0;
  if (t >= 255.f) return 255;
  return (int)t;
}

__device__ __forceinline__ int luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

__device__ __forceinline__ void hue_rotate(int& r, int& g, int& b, int shift) {
  // rgb2hsv_row
  const int mx = max(r, max(g, b)), mn = min(r, min(g, b));
  int uh = 0, us = 0;
  const int v = mx;
  if (mx != mn) {
    const float cr = (float)(mx - mn);
    const float s = __fdiv_rn(cr, (float)mx);
    const float rc = __fdiv_rn((float)(mx - r), cr);
    const float gc = __fdiv_rn((float)(mx - g), cr);
    const float bc = __fdiv_rn((float)(mx - b), cr);
    float h;
    if (r == mx) h = __fsub_rn(bc, gc);
    else if (g == mx) h = __double2float_rn(__dsub_rn(__dadd_rn(2.0, (double)rc), (double)bc));
    else h = __double2float_rn(__dsub_rn(__dadd_rn(4.0, (double)gc), (double)rc));
    h = __double2float_rn(fmod(__dadd_rn(__ddiv_rn((double)h, 6.0), 1.0), 1.0));
    uh = clip8(__double2int_rz(__dmul_rn((double)h, 255.0)));
    us = clip8(__double2int_rz(__dmul_rn((double)s, 255.0)));
  }
  uh = (uh + shift) & 255;
  // hsv2rgb
  if (us == 0) {
    r = g = b = v;
    return;
  }
  const double hd = __ddiv_rn(__dmul_rn((double)uh, 6.0), 255.0);
  const int i = (int)floor(hd);
  const float f = __double2float_rn(__dsub_rn(hd, (double)(float)i));
  const float fs = __double2float_rn(__ddiv_rn((double)us, 255.0));
  const double vv = (double)v;
  const int p = clip8((int)round(__dmul_rn(vv, __dsub_rn(1.0, (double)fs))));
  const int q = clip8((int)round(__dmul_rn(vv, __dsub_rn(1.0, (double)__fmul_rn(fs, f)))));
  const int t = clip8((int)round(__dmul_rn(vv, __dsub_rn(1.0, __dmul_rn((double)fs, __dsub_rn(1.0, (double)f))))));
  switch (i % 6) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

__device__ __forceinline__ void apply_step(int op, const JitterImg& d, int mean, int& r, int& g, int& b) {
  if (op == kBrightness) {
    r = blend1(0, r, d.bright); g = blend1(0, g, d.bright); b = blend1(0, b, d.bright);
  } else if (op == kContrast) {
    r = blend1(mean, r, d.contr); g = blend1(mean, g, d.contr); b = blend1(mean, b, d.contr);
  } else if (op == kSaturation) {
    const int l = luma(r, g, b);
    r = blend1(l, r, d.sat); g = blend1(l, g, d.sat); b = blend1(l, b, d.sat);
  } else {
    hue_rotate(r, g, b, d.hue_shift);
  }
}

// the image whose block range holds `blk` (block0 ascending)
__device__ __forceinline__ int find_image(const JitterImg* imgs, int n, unsigned blk) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (imgs[mid].block0 <= blk) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(kThreads) color_jitter_pre_kernel(uint8_t* buf, const JitterImg* imgs, int n,
                                                                    unsigned long long* lsum) {
  const int im = find_image(imgs, n, blockIdx.x);
  const JitterImg d = imgs[im];
  if (d.n_pre == 0 && !d.contrast) return;
  uint8_t* px = buf + d.off;
  const unsigned long long p0 = (unsigned long long)(blockIdx.x - d.block0) * kPixPerBlock;
  unsigned part = 0;
#pragma unroll
  for (int k = 0; k < kPixPerThread; ++k) {
    const unsigned long long p = p0 + (unsigned long long)k * kThreads + threadIdx.x;
    if (p >= d.npix) break;
    uint8_t* q = px + 3 * p;
    int r = q[0], g = q[1], b = q[2];
    for (int s = 0; s < d.n_pre; ++s) apply_step((d.pre >> 4 * s) & 15, d, 0, r, g, b);
    if (d.n_pre) { q[0] = (uint8_t)r; q[1] = (uint8_t)g; q[2] = (uint8_t)b; }
    part += luma(r, g, b);
  }
  if (!d.contrast) return;
  __shared__ unsigned warp_sum[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long tot = 0;
    for (int w = 0; w < kThreads / 32; ++w) tot += warp_sum[w];
    atomicAdd(lsum + im, tot);
  }
}

__global__ void __launch_bounds__(kThreads) color_jitter_post_kernel(uint8_t* buf, const JitterImg* imgs, int n,
                                                                     const unsigned long long* lsum) {
  const int im = find_image(imgs, n, blockIdx.x);
  const JitterImg d = imgs[im];
  if (!d.contrast) return;
  // ImageStat.Stat(L).mean[0] is sum / count in double; ImageEnhance.Contrast takes int(mean + 0.5)
  const int mean = (int)__dadd_rn(__ddiv_rn((double)lsum[im], (double)d.npix), 0.5);
  uint8_t* px = buf + d.off;
  const unsigned long long p0 = (unsigned long long)(blockIdx.x - d.block0) * kPixPerBlock;
#pragma unroll
  for (int k = 0; k < kPixPerThread; ++k) {
    const unsigned long long p = p0 + (unsigned long long)k * kThreads + threadIdx.x;
    if (p >= d.npix) break;
    uint8_t* q = px + 3 * p;
    int r = q[0], g = q[1], b = q[2];
    apply_step(kContrast, d, mean, r, g, b);
    for (int s = 0; s < d.n_post; ++s) apply_step((d.post >> 4 * s) & 15, d, 0, r, g, b);
    q[0] = (uint8_t)r; q[1] = (uint8_t)g; q[2] = (uint8_t)b;
  }
}

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

}  // namespace

struct JitterWs {
  uint8_t* host = nullptr;   // pinned staging of descriptors + zeroed sums
  size_t host_cap = 0;
  void* dev = nullptr;
  size_t dev_cap = 0;
  cudaEvent_t copied = nullptr;   // the H2D copy out of `host` has finished
  bool pending = false;
  cudaEvent_t done = nullptr;     // the last kernel reading `dev` has finished
  bool used = false;
};

void jitter_ws_destroy(JitterWs* ws) {
  if (!ws) return;
  if (ws->pending) cudaEventSynchronize(ws->copied);
  if (ws->host) cudaFreeHost(ws->host);
  if (ws->dev) cudaFree(ws->dev);
  if (ws->copied) cudaEventDestroy(ws->copied);
  if (ws->done) cudaEventDestroy(ws->done);
  delete ws;
}

int color_jitter_u8(JitterWs** pws, uint8_t* buf, const uint64_t* out_offsets, const int* H, const int* W,
                    const ibl_color_jitter_params* params, int N, cudaStream_t s, uint64_t* launches) {
  std::vector<JitterImg> imgs(N);
  unsigned long long blocks = 0;
  bool any_pre = false, any_post = false;
  for (int n = 0; n < N; ++n) {
    const ibl_color_jitter_params& pr = params[n];
    JitterImg& d = imgs[n];
    memset(&d, 0, sizeof(d));
    int seen = 0;
    for (int k = 0; k < 4; ++k) {
      IBL_REQUIRE(pr.order[k] >= 0 && pr.order[k] < 4 && !(seen >> pr.order[k] & 1), "order is not a permutation of 0..3");
      seen |= 1 << pr.order[k];
    }
    const float f[4] = {pr.brightness, pr.contrast, pr.saturation, pr.hue};
    for (int k = 0; k < 3; ++k) IBL_REQUIRE(isnan(f[k]) || (f[k] >= 0.f && isfinite(f[k])), "negative or infinite factor");
    IBL_REQUIRE(isnan(f[3]) || (f[3] >= -0.5f && f[3] <= 0.5f), "hue factor outside [-0.5, 0.5]");
    d.contrast = !isnan(f[1]);
    bool after = false;             // past the contrast step (never, when contrast is None: one launch does it all)
    for (int k = 0; k < 4; ++k) {
      const int op = pr.order[k];
      if (op == kContrast) after = d.contrast;
      else if (isnan(f[op])) continue;
      else if (after) d.post |= (unsigned)op << 4 * d.n_post++;
      else d.pre |= (unsigned)op << 4 * d.n_pre++;
    }
    d.bright = f[0];
    d.contr = f[1];
    d.sat = f[2];
    d.hue_shift = isnan(f[3]) ? 0 : ((int)((double)f[3] * 255.0)) & 255;
    IBL_REQUIRE(H[n] >= 1 && W[n] >= 1, "empty image");
    d.off = out_offsets[n];
    d.npix = (unsigned long long)H[n] * W[n];
    d.block0 = (unsigned)blocks;
    blocks += (d.npix + kPixPerBlock - 1) / kPixPerBlock;
    any_pre |= d.n_pre > 0 || d.contrast;
    any_post |= d.contrast != 0;
  }
  IBL_REQUIRE(blocks < (1ull << 31), "batch too large");
  if (!any_pre) return IBL_OK;
  if (!*pws) {
    *pws = new (std::nothrow) JitterWs();
    if (!*pws) return IBL_ERR_OOM;
    IBL_CUDA_OK(cudaEventCreateWithFlags(&(*pws)->copied, cudaEventDisableTiming));
    IBL_CUDA_OK(cudaEventCreateWithFlags(&(*pws)->done, cudaEventDisableTiming));
  }
  JitterWs* ws = *pws;
  // staging: descriptors | per-image L sums (zero)
  const size_t o_sum = align16(sizeof(JitterImg) * N), bytes = o_sum + sizeof(unsigned long long) * N;
  if (ws->pending) {                                  // the previous call's H2D copy still reads the pinned buffer
    IBL_CUDA_OK(cudaEventSynchronize(ws->copied));
    ws->pending = false;
  }
  if (ws->host_cap < bytes) {
    if (ws->host) cudaFreeHost(ws->host);
    ws->host = nullptr;
    ws->host_cap = 0;
    if (cudaMallocHost(&ws->host, bytes) != cudaSuccess) {
      cudaGetLastError();
      set_last_error("color jitter staging cudaMallocHost failed");
      return IBL_ERR_OOM;
    }
    ws->host_cap = bytes;
  }
  // the previous call's kernels may still read the device descriptors and sums, possibly on another stream:
  // order this call's copy after them (cudaFree below synchronises the device by itself)
  if (ws->used) IBL_CUDA_OK(cudaStreamWaitEvent(s, ws->done, 0));
  if (ws->dev_cap < bytes) {
    if (ws->dev) cudaFree(ws->dev);
    ws->dev = nullptr;
    ws->dev_cap = 0;
    const cudaError_t e = cudaMalloc(&ws->dev, bytes);
    if (e != cudaSuccess) {
      cudaGetLastError();
      set_last_error("color jitter workspace cudaMalloc(" + std::to_string(bytes) + " B) failed: " + cudaGetErrorString(e));
      return IBL_ERR_OOM;
    }
    ws->dev_cap = bytes;
  }
  memcpy(ws->host, imgs.data(), sizeof(JitterImg) * N);
  memset(ws->host + o_sum, 0, sizeof(unsigned long long) * N);
  IBL_CUDA_OK(cudaMemcpyAsync(ws->dev, ws->host, bytes, cudaMemcpyHostToDevice, s));
  IBL_CUDA_OK(cudaEventRecord(ws->copied, s));
  ws->pending = true;
  const JitterImg* d_imgs = static_cast<const JitterImg*>(ws->dev);
  unsigned long long* d_sum = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(ws->dev) + o_sum);
  color_jitter_pre_kernel<<<(unsigned)blocks, kThreads, 0, s>>>(buf, d_imgs, N, d_sum);
  if (launches) ++*launches;
  if (any_post) {
    color_jitter_post_kernel<<<(unsigned)blocks, kThreads, 0, s>>>(buf, d_imgs, N, d_sum);
    if (launches) ++*launches;
  }
  IBL_CUDA_OK(cudaGetLastError());
  IBL_CUDA_OK(cudaEventRecord(ws->done, s));
  ws->used = true;
  return IBL_OK;
}

}  // namespace ibl
