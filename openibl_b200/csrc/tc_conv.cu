// 3x3 / stride 1 / pad 1 convolution as a Hopper wgmma implicit GEMM (reference: the 12 convs
// conv1_2..conv5_3 of ibl/models/vgg.py:40-42,61-62, cuDNN in the reference).
//
//   M = output pixels (128 per tile: TH x TW patch of one image)
//   N = output channels (BN per tile)
//   K = 9 taps x Cin, walked as (tap, 64-channel chunk)
//
// fp32 parity on a tensor core without an fp32 mode: every fp32 operand is carried as two bf16
// planes (hi = bf16(x), lo = bf16(x - hi)) and each K-chunk issues three MMAs
//   A_lo.B_hi + A_hi.B_lo + A_hi.B_hi      (fp32 accumulation in registers),
// dropping only the lo.lo term (~2^-16 relative).  Activations live in HBM as NHWC bf16 hi/lo
// planes, weights as [tap][Cout][Cin] hi/lo planes, so every operand tile is one TMA box:
// the activation box for tap (kh,kw) is the output patch shifted by (kh-1,kw-1) and the
// hardware zero-fills the out-of-image part, which is exactly the conv's zero padding.
//
// Warp roles, persistent over tiles.  Box staging (BN = 64, 160 threads):
//   warps 0-3  consumer warpgroup: wgmma main loop (two m64 halves of the 128-pixel tile), then the epilogue
//   warp 4     TMA producer
// Halo staging (BN = 128, 384 threads, "ping-pong"):
//   warpgroup 0     producer (warp 0 issues the TMA loads), its registers handed to the consumers (setmaxnreg)
//   warpgroups 1-2  consumers: consumer j takes the CTA's tiles j, j+2, j+4, ... so one runs its epilogue while the
//                   other issues the next tile's MMAs
// Epilogue: accumulator -> row-per-thread views (Acc128::rows32), + bias, ReLU, optional fused 2x2 max-pool
// (warp shuffles), split into hi/lo planes (or fp32 for conv5_3), 16-byte stores.
//
// Wide tiles (WTW = 16: 16x16 patches of 256 pixels, the same 384-thread halo staging and ping-pong consumers) swap
// the operand roles:
//   M = 64 output channels per tile, A = the weights, loaded into registers by ldmatrix once per k16 step
//   N = the 256 pixels, B = two n128 views of the halo tile (patch columns 0-7 and 8-15 of all 16 rows), 8-pixel
//       groups one 18-pixel halo row (2304 B) apart, the second view 8 rows in
// so each weight fragment serves 256 pixels and the pixels are the only operand the tensor core reads from shared
// memory.  A thread then holds both pixels of every horizontal and vertical pool pair, so the epilogue is register-local
// up to one 4-lane transpose per 4 pixels for the NHWC 16-byte stores (conv_wide_epilogue).  (An 8x32 patch, read as
// four n64 views, tiles 120x160 exactly but measured no faster there than the 128-pixel kernel: DESIGN 5, K1b.)
#include "common.cuh"
#include "tc_common.cuh"

namespace ibl {

using namespace tc;

// ---- host: driver entry point ---------------------------------------------------------------
namespace tc {
EncodeTiledFn get_encode_tiled() {
  // initialised exactly once even when several host threads (nn.DataParallel replicas, one per GPU) make their
  // first call together: a plain "tried" flag could let a second thread see the flag before the pointer was stored
  static const EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      return reinterpret_cast<EncodeTiledFn>(p);
    return nullptr;
  }();
  return fn;
}

int make_tmap(CUtensorMap* out, CUtensorMapDataType dt, int rank, const void* base,
              const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) {
    set_last_error("cuTensorMapEncodeTiled is not available (no CUDA driver?)");
    return IBL_ERR_NO_DEVICE;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = enc(out, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return IBL_ERR_CUDA;
  }
  return IBL_OK;
}
}  // namespace tc

int tc_driver_init() { return get_encode_tiled() ? IBL_OK : IBL_ERR_NO_DEVICE; }

// ---- kernel ---------------------------------------------------------------------------------
struct ConvTcArgs {
  int N, H, W, cin, cout;
  int tw_log2;            // TW = 1 << tw_log2 (8 or 16), TH = pixels per tile / TW
  int tiles_w, tiles_h;   // patches per image
  int n_tiles;            // cout / BN
  int total_tiles;        // N * tiles_h * tiles_w * n_tiles
  int relu, pool;
  const float* bias;
  __nv_bfloat16* y_hi;
  __nv_bfloat16* y_lo;
  float* y_f32;
  float* ssq;             // optional [n_tiles][N*H*W] per-pixel sum of squares of the outputs (no pool)
  long long ssq_stride;
};

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// One accumulator tile (128 pixel rows x BN output channels, thread = pixel row (r, c) of the patch) to global memory:
// bias + ReLU + fused 2x2 max-pool + bf16 hi/lo split (or fp32), optional per-pixel sum of squares.  `dr_lanes` is the
// lane distance between a pixel and the one below it; `bar` is the warpgroup's named barrier.
template <int BN>
__device__ __forceinline__ void conv_epilogue_tile(const ConvTcArgs& a, const Acc128<BN>& acc, float* stg, int img, int h0,
                                                   int w0, int n0, int nt, int r, int c, int dr_lanes, int bar = 1) {
  const int h = h0 + r, w = w0 + c;
  bool valid;
  long long pix;
  if (a.pool) {
    const int OH = a.H >> 1, OW = a.W >> 1;
    const int oh = h >> 1, ow = w >> 1;
    valid = oh < OH && ow < OW && img < a.N;      // all four lanes of a window store (8 channels each per 32-channel chunk)
    pix = ((long long)img * OH + oh) * OW + ow;
  } else {
    valid = h < a.H && w < a.W && img < a.N;
    pix = ((long long)img * a.H + h) * a.W + w;
  }
  float ssq_acc = 0.f;   // per-pixel sum of squares over this N tile (feeds NetVLAD's input norm)
#pragma unroll
  for (int ch = 0; ch < BN / 32; ++ch) {     // unrolled: the accumulator is indexed with constants only
    uint32_t raw[32];
    acc.rows32(ch, stg, raw, bar);
    if (a.pool) {
      // 2x2 max-pool BEFORE bias / ReLU / split (. + b and max(., 0) are monotone, so the results are the same bits)
      // as a two-step exchange: against the w-neighbour (lane ^ 1) every lane keeps one half of the 32
      // channels and sends the other, against the h-neighbour (lane ^ dr_lanes) one half of those 16 -- 24 shuffles instead
      // of 64, and each of the window's four lanes finishes 8 channels (bias, ReLU, hi/lo, ONE 16-byte store per plane)
      // instead of one lane doing all 32 while three idle.
      const bool s1 = (c & 1) != 0, s2 = (r & 1) != 0;
      float u[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float lo_h = __uint_as_float(raw[j]), hi_h = __uint_as_float(raw[j + 16]);
        const float got = __shfl_xor_sync(0xffffffffu, s1 ? lo_h : hi_h, 1);
        u[j] = fmaxf(s1 ? hi_h : lo_h, got);
      }
      float w8[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float got = __shfl_xor_sync(0xffffffffu, s2 ? u[j] : u[j + 8], dr_lanes);
        w8[j] = fmaxf(s2 ? u[j + 8] : u[j], got);
      }
      if (valid) {
        const int cbase = n0 + ch * 32 + (s1 ? 16 : 0) + (s2 ? 8 : 0);
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(a.bias + cbase));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(a.bias + cbase) + 1);
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          w8[j] = w8[j] + bb[j];
          if (a.relu) w8[j] = fmaxf(w8[j], 0.f);
        }
        const long long off = pix * a.cout + cbase;
        if (a.y_f32) {
          float4* o = reinterpret_cast<float4*>(a.y_f32 + off);
          o[0] = make_float4(w8[0], w8[1], w8[2], w8[3]);
          o[1] = make_float4(w8[4], w8[5], w8[6], w8[7]);
        } else {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float x0 = w8[2 * j], x1 = w8[2 * j + 1];
            const __nv_bfloat16 h0b = __float2bfloat16_rn(x0), h1b = __float2bfloat16_rn(x1);
            __nv_bfloat162 hh(h0b, h1b);
            hi[j] = *reinterpret_cast<uint32_t*>(&hh);
            lo[j] = pack_bf16x2(x0 - __bfloat162float(h0b), x1 - __bfloat162float(h1b));
          }
          *reinterpret_cast<uint4*>(a.y_hi + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          *reinterpret_cast<uint4*>(a.y_lo + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
      }
      continue;
    }
    float v[32];
    const float4* bp = reinterpret_cast<const float4*>(a.bias + n0 + ch * 32);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 b = __ldg(bp + j);
      v[4 * j + 0] = __uint_as_float(raw[4 * j + 0]) + b.x;
      v[4 * j + 1] = __uint_as_float(raw[4 * j + 1]) + b.y;
      v[4 * j + 2] = __uint_as_float(raw[4 * j + 2]) + b.z;
      v[4 * j + 3] = __uint_as_float(raw[4 * j + 3]) + b.w;
    }
    if (a.relu) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
    }
    if (a.ssq) {
#pragma unroll
      for (int j = 0; j < 32; ++j) ssq_acc = fmaf(v[j], v[j], ssq_acc);
    }
    if (valid) {
      const long long off = pix * a.cout + n0 + ch * 32;
      if (a.y_f32) {
        float4* o = reinterpret_cast<float4*>(a.y_f32 + off);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
      } else {
        uint32_t hi[16], lo[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float x0 = v[2 * j], x1 = v[2 * j + 1];
          const __nv_bfloat16 h0b = __float2bfloat16_rn(x0), h1b = __float2bfloat16_rn(x1);
          __nv_bfloat162 hh(h0b, h1b);
          hi[j] = *reinterpret_cast<uint32_t*>(&hh);
          lo[j] = pack_bf16x2(x0 - __bfloat162float(h0b), x1 - __bfloat162float(h1b));
        }
        uint4* oh4 = reinterpret_cast<uint4*>(a.y_hi + off);
        uint4* ol4 = reinterpret_cast<uint4*>(a.y_lo + off);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          oh4[j] = make_uint4(hi[4 * j], hi[4 * j + 1], hi[4 * j + 2], hi[4 * j + 3]);
          ol4[j] = make_uint4(lo[4 * j], lo[4 * j + 1], lo[4 * j + 2], lo[4 * j + 3]);
        }
      }
    }
  }
  if (a.ssq && valid && !a.pool) a.ssq[(long long)nt * a.ssq_stride + pix] = ssq_acc;
}

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;                       // bf16 elements per K-chunk = one 128-byte row
constexpr int TC_A_BYTES = TC_BM * TC_BK * 2;   // 16 KiB per plane

// HALO: instead of one [128 px][64 ch] im2col box per tap, the producer stages ONE halo tile per 64-channel
// chunk -- the (16+2) x (8+2) pixel neighbourhood of a 16x8 patch, 180 rows of 128 B per plane -- and the
// nine taps are nine views of it: tap (kh,kw) starts (kh*10 + kw) rows into the tile and consecutive 8-pixel
// row groups are 10 rows (1280 B) apart.  The 128B swizzle is a function of the shared-memory address, so a
// descriptor whose start is only 128-byte aligned and whose group stride is not a multiple of 1024 B reads the
// TMA-written tile correctly (pinned on hardware by tests/test_gpu_parity.py through tc_probe.cu).
// L2->SM traffic of the A operand drops from 9 x 32 KiB to 45 KiB per chunk; the weights get their own ring.
// An 8x16 patch (chosen where it wastes fewer rows, e.g. 120x160 maps) has an 18 x 10 halo: the same 180 rows, taps
// (kh*18 + kw) rows in, 8-row groups 18 rows (2304 B) apart, and the second m64 half (columns 8-15 of every patch row)
// 8 rows in.
constexpr int TC_HALO_W = 10, TC_HALO_H = 18;   // the 16x8 patch's halo
constexpr int TC_HALO_ROWS = TC_HALO_W * TC_HALO_H;
constexpr int TC_HALO_PLANE = 23 * 1024;        // 180 rows x 128 B = 23040 B, padded to the swizzle period

// The wide tiles' halo: (16+2) x (16+2) = 324 rows of 128 B per plane, padded to the swizzle period.  Two stages of both
// planes and three 16 KiB weight taps leave no room for epilogue staging.
constexpr int TC_WIDE_PX = 256;
constexpr int TC_WIDE_HALO_PLANE = 41 * 1024;

template <int BN, int STAGES, bool HALO = false, int NA = 0, int WTW = 0>
struct ConvTcSmem {
  static constexpr int THREADS = HALO ? 384 : 160;
  static constexpr int CONSUMERS = HALO ? 2 : 1;   // consumer warpgroups, each with its own epilogue staging buffer
  static constexpr int B_BYTES = BN * TC_BK * 2;
  static constexpr int STAGE_BYTES = HALO ? 2 * B_BYTES : 2 * TC_A_BYTES + 2 * B_BYTES;
  static constexpr int HALO_PLANE = WTW ? TC_WIDE_HALO_PLANE : TC_HALO_PLANE;
  static constexpr int A_RING = HALO ? NA * 2 * HALO_PLANE : 0;
  static constexpr int STG = WTW ? 0 : CONSUMERS * ACC_STG_BYTES;
  static constexpr int BYTES = A_RING + STAGES * STAGE_BYTES + STG + 1024 /*align slack*/ + 256 /*barriers*/;
};

// One wide tile's accumulator: 64 output channels x 256 pixels as two n128 fragments, one per view.  Thread t (warp w,
// lane l) holds in view v, for patch row i: [4i + e] = pixel (i, 8v + 2(l%4) + (e & 1)) of the channel that accumulator
// row 16w + l/4 + 8(e >> 1) stands for (see the weight row map in the kernel).
struct AccWide {
  float d[2][64];
};

__device__ __forceinline__ float wide_pick(bool swap, float a, float b) { return swap ? b : a; }

// In-place transpose of x[4][2] across the four lanes l, l ^ 4, l ^ 8, l ^ 12 (index j = (l >> 2) & 3): afterwards lane j
// holds in x[p] what lane p held in x[j].
__device__ __forceinline__ void wide_transpose4(uint32_t (&x)[4][2], int j) {
#pragma unroll
  for (int bit = 0; bit < 2; ++bit) {
    const bool mine = ((j >> bit) & 1) != 0;
#pragma unroll
    for (int p0 = 0; p0 < 4; ++p0) {
      if (p0 & (1 << bit)) continue;
      const int p1 = p0 | (1 << bit);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t got = __shfl_xor_sync(0xffffffffu, mine ? x[p0][h] : x[p1][h], 4 << bit);
        if (mine) x[p0][h] = got; else x[p1][h] = got;
      }
    }
  }
}

// Wide tile -> global memory: bias + ReLU + fused 2x2 max-pool + bf16 hi/lo split (or fp32), optional per-pixel sum of
// squares (one partial per warp: 16 channels).  The thread's two accumulator rows are the adjacent channels
// c = n0 + 16w + 2(l/4) and c + 1; four pixels at a time go through wide_transpose4, after which lane l stores the 8
// channels n0 + 16w + 8((l >> 4) & 1) .. + 7 of pixel ((l >> 2) & 3) of the four as one 16-byte word per plane.
__device__ __forceinline__ void conv_wide_epilogue(const ConvTcArgs& a, const AccWide& acc, int img, int h0, int w0,
                                                   int nt) {
  constexpr int NV = 2, TH = 16;
  const int t = threadIdx.x & 127, w = t >> 5, lane = t & 31, g = lane >> 2, q = lane & 3, j = g & 3;
  const bool sw = (g >> 2) != 0;                 // rows 16w + g / + 8 are channels c + 1 / c (not c / c + 1)
  const int c = nt * 64 + 16 * w + 2 * g;
  const int cst = nt * 64 + 16 * w + 8 * (g >> 2);   // first of the 8 channels this lane stores
  const float b0 = __ldg(a.bias + c), b1 = __ldg(a.bias + c + 1);
  auto activate = [&](float& v0, float& v1) {
    v0 += b0; v1 += b1;
    if (a.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
  };
  auto pack = [&](float v0, float v1, uint32_t (&x)[2]) {
    if (a.y_f32) {
      x[0] = __float_as_uint(v0); x[1] = __float_as_uint(v1);
    } else {
      const __nv_bfloat16 h0b = __float2bfloat16_rn(v0), h1b = __float2bfloat16_rn(v1);
      __nv_bfloat162 hh(h0b, h1b);
      x[0] = *reinterpret_cast<uint32_t*>(&hh);
      x[1] = pack_bf16x2(v0 - __bfloat162float(h0b), v1 - __bfloat162float(h1b));
    }
  };
  auto store = [&](const uint32_t (&x)[4][2], bool valid, long long pix) {
    if (!valid) return;
    const long long off = pix * a.cout + cst;
    if (a.y_f32) {
      float4* o = reinterpret_cast<float4*>(a.y_f32 + off);
      o[0] = make_float4(__uint_as_float(x[0][0]), __uint_as_float(x[0][1]), __uint_as_float(x[1][0]), __uint_as_float(x[1][1]));
      o[1] = make_float4(__uint_as_float(x[2][0]), __uint_as_float(x[2][1]), __uint_as_float(x[3][0]), __uint_as_float(x[3][1]));
    } else {
      *reinterpret_cast<uint4*>(a.y_hi + off) = make_uint4(x[0][0], x[1][0], x[2][0], x[3][0]);
      *reinterpret_cast<uint4*>(a.y_lo + off) = make_uint4(x[0][1], x[1][1], x[2][1], x[3][1]);
    }
  };
  if (a.pool) {
    // 2x2 max-pool BEFORE bias / ReLU / split, as conv_epilogue_tile: window (b, v) = patch rows 2b, 2b + 1 and columns
    // 8v + 2q, + 1, all four pixels in this thread; four windows b = 4m .. 4m + 3 per transpose
    const int OH = a.H >> 1, OW = a.W >> 1;
    const int ow = (w0 >> 1) + q;   // window column of view 0
#pragma unroll
    for (int v = 0; v < NV; ++v)
#pragma unroll
      for (int m = 0; m < TH / 8; ++m) {
        uint32_t x[4][2];
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float* r0 = &acc.d[v][4 * (2 * (4 * m + p))];
          const float* r1 = r0 + 4;
          const float e0 = fmaxf(fmaxf(r0[0], r0[1]), fmaxf(r1[0], r1[1]));   // accumulator row 16w + g
          const float e1 = fmaxf(fmaxf(r0[2], r0[3]), fmaxf(r1[2], r1[3]));   // row 16w + g + 8
          float v0 = wide_pick(sw, e0, e1), v1 = wide_pick(sw, e1, e0);
          activate(v0, v1);
          pack(v0, v1, x[p]);
        }
        wide_transpose4(x, j);
        const int oh = (h0 >> 1) + 4 * m + j, owv = ow + 4 * v;
        store(x, oh < OH && owv < OW && img < a.N, ((long long)img * OH + oh) * OW + owv);
      }
    return;
  }
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int b = 0; b < TH / 2; ++b) {
      // pixels p = (patch row 2b + (p >> 1), column 8v + 2q + (p & 1))
      uint32_t x[4][2];
      float sq[4];
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const float* r = &acc.d[v][4 * (2 * b + (p >> 1)) + (p & 1)];
        const float e0 = r[0], e1 = r[2];
        float v0 = wide_pick(sw, e0, e1), v1 = wide_pick(sw, e1, e0);
        activate(v0, v1);
        sq[p] = fmaf(v1, v1, v0 * v0);
        pack(v0, v1, x[p]);
      }
      wide_transpose4(x, j);
      const int h = h0 + 2 * b + (j >> 1), wc = w0 + 8 * v + 2 * q + (j & 1);
      const bool valid = h < a.H && wc < a.W && img < a.N;
      const long long pix = ((long long)img * a.H + h) * a.W + wc;
      store(x, valid, pix);
      if (a.ssq) {
        // |x|^2 over the warp's 16 channels: the eight lanes of a pixel column (l ^ 4, l ^ 8, l ^ 16), in a fixed order
        float mine = 0.f;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          float s2 = sq[p];
          s2 += __shfl_xor_sync(0xffffffffu, s2, 4);
          s2 += __shfl_xor_sync(0xffffffffu, s2, 8);
          s2 += __shfl_xor_sync(0xffffffffu, s2, 16);
          if (p == j) mine = s2;
        }
        if (valid && g < 4) a.ssq[(long long)(nt * 4 + w) * a.ssq_stride + pix] = mine;
      }
    }
}

template <int BN, int STAGES, bool HALO, int NA, int WTW = 0>
__global__ void __launch_bounds__(ConvTcSmem<BN, STAGES, HALO, NA, WTW>::THREADS, 1)
conv3x3_tc_kernel(const __grid_constant__ CUtensorMap tm_xhi, const __grid_constant__ CUtensorMap tm_xlo,
                  const __grid_constant__ CUtensorMap tm_whi, const __grid_constant__ CUtensorMap tm_wlo,
                  const ConvTcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle; dynamic smem base is only 16B-aligned
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  using L = ConvTcSmem<BN, STAGES, HALO, NA, WTW>;
  constexpr int HALO_PLANE = L::HALO_PLANE;
  constexpr int HALO_STAGE = 2 * HALO_PLANE;
  constexpr int PX = WTW ? TC_WIDE_PX : TC_BM;   // pixels per tile
  constexpr int B_BYTES = L::B_BYTES;
  constexpr int STAGE_BYTES = L::STAGE_BYTES;
  constexpr int A_RING = L::A_RING;           // HALO: the halo ring sits in front of the weight ring
  uint8_t* ring = smem + A_RING;
  float* stg = reinterpret_cast<float*>(ring + STAGES * STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + STAGES * STAGE_BYTES + L::STG);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* afull_bar = bars + 2 * STAGES;    // HALO only: [NA] + [NA] + the two consumers' order barriers
  uint64_t* aempty_bar = afull_bar + NA;
  uint64_t* order_bar = aempty_bar + NA;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int worker = (int)blockIdx.x;
  const int n_workers = (int)gridDim.x;
  const int producer_warp = HALO ? 0 : 4;
  if (warp == producer_warp && lane == 0) {
    tma_prefetch_desc(&tm_xhi);
    tma_prefetch_desc(&tm_xlo);
    tma_prefetch_desc(&tm_whi);
    tma_prefetch_desc(&tm_wlo);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);   // one arrival per warp of the consuming warpgroup
    }
    for (int i = 0; i < NA; ++i) {
      mbar_init(&afull_bar[i], 1);
      mbar_init(&aempty_bar[i], 4);
    }
    if (HALO) {
      mbar_init(&order_bar[0], 4);
      mbar_init(&order_bar[1], 4);
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  const int TW = 1 << a.tw_log2;
  const int kchunks = a.cin / TC_BK;
  const int kiters = 9 * kchunks;
  const int tiles_per_img = a.tiles_h * a.tiles_w;
  auto coords = [&](int tile, int& img, int& h0, int& w0, int& nt) {
    nt = tile % a.n_tiles;
    const int pt = tile / a.n_tiles;
    img = pt / tiles_per_img;
    const int rem = pt - img * tiles_per_img;
    h0 = (rem / a.tiles_w) * (PX >> a.tw_log2);
    w0 = (rem % a.tiles_w) * TW;
  };

  if (HALO && warp < 4) setmaxnreg_dec<40>();
  if (warp == producer_warp) {
    // ================= TMA producer: convergent warp, one elected lane issues, coordinates warp-uniform =================
    const uint32_t smem_a = warp_uniform(smem_u32(smem));
    const uint32_t ring_a = smem_a + A_RING;
    const uint32_t bars_a = ring_a + STAGES * STAGE_BYTES + L::STG;
    const uint32_t full_a = bars_a, empty_a = bars_a + 8 * STAGES;
    const uint32_t afull_a = bars_a + 16 * STAGES, aempty_a = afull_a + 8 * NA;
    // the two weight planes of one tap (into `st`, planes B_BYTES apart)
    auto load_w = [&](uint32_t st, uint32_t fb, int c0, int n0, int tap) {
      tma_load_3d_a(st, &tm_whi, fb, c0, n0, tap);
      tma_load_3d_a(st + B_BYTES, &tm_wlo, fb, c0, n0, tap);
    };
    int stage = 0;
    uint32_t phase = 0;
    if constexpr (HALO) {
      // Two independent streams -- halo tiles (one per tile and 64-channel chunk) and weight taps (nine per halo) --
      // each issued as soon as its ring has a free slot, so the halo of the NEXT chunk is in flight while the taps of
      // the current one are still being fed.  Lane 0 polls once; the answer is broadcast so that the branch on it is
      // warp-uniform.
      auto try_wait_warp = [&](uint32_t bar, uint32_t parity) -> bool {
        uint32_t ok = 0;
        if (lane == 0) {
          asm volatile(
              "{\n\t"
              ".reg .pred p;\n\t"
              "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
              "selp.u32 %0, 1, 0, p;\n\t"
              "}"
              : "=r"(ok)
              : "r"(bar), "r"(parity)
              : "memory");
        }
        return warp_uniform(ok) != 0;
      };
      int astage = 0;
      uint32_t aphase = 0;
      int tA = worker, kcA = 0, tB = worker, kcB = 0, tapB = 0;
      while (tB < a.total_tiles) {
        const uint32_t as_u = warp_uniform((uint32_t)astage);
        if (tA < a.total_tiles && try_wait_warp(aempty_a + 8 * as_u, aphase ^ 1)) {
          int img, h0, w0, nt;
          coords(tA, img, h0, w0, nt);
          img = (int)warp_uniform((uint32_t)img); h0 = (int)warp_uniform((uint32_t)h0);
          w0 = (int)warp_uniform((uint32_t)w0);
          const int c0 = (int)warp_uniform((uint32_t)(kcA * TC_BK));
          const uint32_t sa = smem_a + as_u * HALO_STAGE;
          constexpr uint32_t kHaloBytes = WTW ? 2u * (WTW + 2) * (TC_WIDE_PX / WTW + 2) * 128u : 2u * TC_HALO_ROWS * 128u;
          if (elect_one()) {
            mbar_arrive_expect_tx_a(afull_a + 8 * as_u, kHaloBytes);
            tma_load_4d_a(sa, &tm_xhi, afull_a + 8 * as_u, c0, w0 - 1, h0 - 1, img);
            tma_load_4d_a(sa + HALO_PLANE, &tm_xlo, afull_a + 8 * as_u, c0, w0 - 1, h0 - 1, img);
          }
          __syncwarp();
          if (++astage == NA) { astage = 0; aphase ^= 1; }
          if (++kcA == kchunks) { kcA = 0; tA += n_workers; }
          continue;
        }
        const uint32_t st_u = warp_uniform((uint32_t)stage);
        if (try_wait_warp(empty_a + 8 * st_u, phase ^ 1)) {
          int img, h0, w0, nt;
          coords(tB, img, h0, w0, nt);
          const int n0 = (int)warp_uniform((uint32_t)(nt * BN));
          const int c0 = (int)warp_uniform((uint32_t)(kcB * TC_BK));
          const int tap = (int)warp_uniform((uint32_t)tapB);
          const uint32_t st = ring_a + st_u * STAGE_BYTES;
          if (elect_one()) {
            mbar_arrive_expect_tx_a(full_a + 8 * st_u, STAGE_BYTES);
            load_w(st, full_a + 8 * st_u, c0, n0, tap);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
          if (++tapB == 9) { tapB = 0; if (++kcB == kchunks) { kcB = 0; tB += n_workers; } }
        }
      }
    } else
    for (int tile = worker; tile < a.total_tiles; tile += n_workers) {
      int img, h0, w0, nt;
      coords(tile, img, h0, w0, nt);
      img = (int)warp_uniform((uint32_t)img); h0 = (int)warp_uniform((uint32_t)h0);
      w0 = (int)warp_uniform((uint32_t)w0);
      const int n0 = (int)warp_uniform((uint32_t)(nt * BN));
      for (int kit = 0; kit < kiters; ++kit) {
        const int tap = (int)warp_uniform((uint32_t)(kit / kchunks));
        const int c0 = (int)warp_uniform((uint32_t)((kit - tap * kchunks) * TC_BK));
        const int kh = tap / 3 - 1, kw = tap % 3 - 1;
        const uint32_t st_u = warp_uniform((uint32_t)stage);
        mbar_wait_warp_a(empty_a + 8 * st_u, phase ^ 1);
        const uint32_t st = smem_a + st_u * STAGE_BYTES;
        if (elect_one()) {
          const uint32_t fb = full_a + 8 * st_u;
          mbar_arrive_expect_tx_a(fb, STAGE_BYTES);
          tma_load_4d_a(st, &tm_xhi, fb, c0, w0 + kw, h0 + kh, img);
          tma_load_4d_a(st + TC_A_BYTES, &tm_xlo, fb, c0, w0 + kw, h0 + kh, img);
          load_w(st + 2 * TC_A_BYTES, fb, c0, n0, tap);
        }
        __syncwarp();
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (!HALO || warp >= 4) {
    const uint32_t smem_a = smem_u32(smem);
    const uint32_t ring_a = smem_a + A_RING;
    auto release_w = [&](int st) {          // this warp is done reading weight slot st
      if (lane == 0) mbar_arrive(&empty_bar[st]);
    };
    if constexpr (WTW != 0) {
    // ================= wide tiles: two consumer warpgroups (ping-pong), weights in registers =================
    setmaxnreg_inc<232>();
    static_assert(WTW == 16, "the wide tiles are 16x16 patches");
    constexpr int NV = 2;                         // n128 pixel views per tap
    const int cw = warp / 4 - 1;
    // Weight row map: accumulator rows 16w + j and 16w + j + 8 (j < 8) read output channels 16w + 2j + s and
    // 16w + 2j + (s ^ 1), s = j >> 2: a thread's two rows are adjacent channels, and the eight rows of each ldmatrix
    // phase fall on eight distinct 128B-swizzle phases (no bank conflicts).  Lane l addresses row 16w + (l & 7) + 8 bit3(l).
    const int wq = (threadIdx.x >> 5) & 3, jl = lane & 7, hl = (lane >> 3) & 1;
    const int wrow = 16 * wq + 2 * jl + (hl ^ (jl >> 2));
    const uint32_t halo_w = (uint32_t)WTW + 2;     // halo row pitch (pixels): the views' 8-pixel group stride
    const uint64_t halo_desc = ((uint64_t)1 << 16) | ((uint64_t)((halo_w * 128) >> 4) << 32) | ((uint64_t)1 << 62);
    // Ring arithmetic and order barrier as in the 128-pixel halo kernel below.
    for (int i = cw; worker + i * n_workers < a.total_tiles; i += 2) {
      int img, h0, w0, nt;
      coords(worker + i * n_workers, img, h0, w0, nt);
      int astage = (i * kchunks) % NA, stage = (i * kiters) % STAGES;
      uint32_t aphase = (uint32_t)((i * kchunks) / NA) & 1u, phase = (uint32_t)((i * kiters) / STAGES) & 1u;
      if (i > 0) mbar_wait(&order_bar[cw], (uint32_t)((i - 1) >> 1) & 1u);
      AccWide acc;
      int prev = -1, prev_a = -1, kc = 0, tap = 0;
      // The weight fragments of one k16 step go into f[k & 1] while the previous step's MMAs run: 16 registers next to
      // the 128 of the accumulator (the kernel is compiled for 168).
      uint32_t f[2][2][4];
      for (int kit = 0; kit < kiters; ++kit) {
        if (tap == 0) mbar_wait(&afull_bar[astage], aphase);
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sb = ring_a + stage * STAGE_BYTES;
        ldsm_a_sw128(f[0][0], sb, wrow, 0);
        ldsm_a_sw128(f[0][1], sb + B_BYTES, wrow, 0);
        const uint32_t ha = smem_a + astage * HALO_STAGE;
        const uint32_t toff = ((uint32_t)(tap / 3) * halo_w + (uint32_t)(tap % 3)) * 128u;
        const uint64_t x_hi = halo_desc | (uint64_t)(((ha + toff) >> 4) & 0x3fffu);
        const uint64_t x_lo = halo_desc | (uint64_t)(((ha + HALO_PLANE + toff) >> 4) & 0x3fffu);
        const uint32_t acc0 = (kc > 0 || tap > 0) ? 1u : 0u;
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) {
          const uint32_t(&fh)[4] = f[k & 1][0];
          const uint32_t(&fl)[4] = f[k & 1][1];
          const uint64_t ko = (uint64_t)(k * 2);
          wgmma_fence();
          // view v starts 8v pixels into patch row 0: +1 KiB
#pragma unroll
          for (int v = 0; v < NV; ++v) WgmmaRS<256 / NV>::mma(acc.d[v], fh, x_lo + 64 * v + ko, (acc0 | k) ? 1u : 0u);
#pragma unroll
          for (int v = 0; v < NV; ++v) WgmmaRS<256 / NV>::mma(acc.d[v], fl, x_hi + 64 * v + ko, 1u);
#pragma unroll
          for (int v = 0; v < NV; ++v) WgmmaRS<256 / NV>::mma(acc.d[v], fh, x_hi + 64 * v + ko, 1u);
          wgmma_commit();
          if (k == 3 && kc == kchunks - 1 && tap == 8 && lane == 0) mbar_arrive(&order_bar[cw ^ 1]);
          wgmma_wait<1>();                    // the previous k16 step's MMAs have retired: its fragments are free
          if (k == 0) {                       // ... and the previous tap's weight slot, and after the first tap of a
            if (prev >= 0) release_w(prev);   // chunk the previous chunk's halo slot
            if (prev_a >= 0) {
              if (lane == 0) mbar_arrive(&aempty_bar[prev_a]);
              prev_a = -1;
            }
          }
          if (k + 1 < TC_BK / 16) {
            ldsm_a_sw128(f[(k + 1) & 1][0], sb, wrow, k + 1);
            ldsm_a_sw128(f[(k + 1) & 1][1], sb + B_BYTES, wrow, k + 1);
          }
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
        if (++tap == 9) {
          tap = 0;
          ++kc;
          prev_a = astage;
          if (++astage == NA) { astage = 0; aphase ^= 1; }
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int v = 0; v < NV; ++v)
#pragma unroll
        for (int e = 0; e < 128 / NV; ++e) asm volatile("" : "+f"(acc.d[v][e])::"memory");
      release_w(prev);
      if (lane == 0) mbar_arrive(&aempty_bar[prev_a]);
      conv_wide_epilogue(a, acc, img, h0, w0, nt);
    }
    } else if constexpr (HALO) {
    // ================= two consumer warpgroups (ping-pong): main loop + epilogue =================
    setmaxnreg_inc<232>();
    const int cw = warp / 4 - 1;            // consumer 0 / 1
    const int bar = 1 + cw;                 // its named barrier (epilogue staging)
    float* my_stg = stg + cw * (ACC_STG_BYTES / 4);
    // accumulator row m -> patch pixel (r, c).  16x8: 8-row group g = pixel row g.  8x16: rows 0-63 are columns 0-7
    // and rows 64-127 columns 8-15 of patch rows 0-7.  Either way the pixel below is 8 rows (lanes) further on.
    const int m = threadIdx.x & 127;
    const int r = TW == 16 ? (m >> 3) & 7 : m >> 3;
    const int c = TW == 16 ? ((m >> 6) << 3) | (m & 7) : m & 7;
    // K-major SW128 view of the halo tile: 8-pixel row groups one halo row (TW + 2 pixels) apart
    const uint32_t halo_w = (uint32_t)TW + 2;
    const uint64_t halo_desc = ((uint64_t)1 << 16) | ((uint64_t)((halo_w * 128) >> 4) << 32) | ((uint64_t)1 << 62);
    const uint64_t a_half = (TW == 16 ? 8u : 8u * halo_w) * 128u / 16u;
    // Consumer cw takes the CTA's tiles cw, cw + 2, ...  The producer fills both rings in tile order, so the slots
    // (and phases) of CTA-local tile i start at running index i * kchunks (halo) and i * kiters (weights).  The order
    // barrier lets a consumer wait on its first slots only after the other consumer has waited on all the slots of
    // the tile before: a slot's full barrier is then at most one phase behind the awaited one, so its parity is exact.
    for (int i = cw; worker + i * n_workers < a.total_tiles; i += 2) {
      int img, h0, w0, nt;
      coords(worker + i * n_workers, img, h0, w0, nt);
      int astage = (i * kchunks) % NA, stage = (i * kiters) % STAGES;
      uint32_t aphase = (uint32_t)((i * kchunks) / NA) & 1u, phase = (uint32_t)((i * kiters) / STAGES) & 1u;
      if (i > 0) mbar_wait(&order_bar[cw], (uint32_t)((i - 1) >> 1) & 1u);
      Acc128<BN> acc;
      int prev = -1, prev_a = -1;
      for (int kc = 0; kc < kchunks; ++kc) {
        mbar_wait(&afull_bar[astage], aphase);
        const uint32_t ha = smem_a + astage * HALO_STAGE;
        for (int tap = 0; tap < 9; ++tap) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t toff = ((uint32_t)(tap / 3) * halo_w + (uint32_t)(tap % 3)) * 128u;
          const uint64_t a_hi = halo_desc | (uint64_t)(((ha + toff) >> 4) & 0x3fffu);
          const uint64_t a_lo = halo_desc | (uint64_t)(((ha + TC_HALO_PLANE + toff) >> 4) & 0x3fffu);
          const uint32_t sb = ring_a + stage * STAGE_BYTES;
          const uint64_t b_hi = gmma_desc_kmajor_sw128(sb), b_lo = gmma_desc_kmajor_sw128(sb + B_BYTES);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < TC_BK / 16; ++k) {
            const uint64_t ko = (uint64_t)(k * 2);
            acc.mma(a_lo + ko, a_lo + a_half + ko, b_hi + ko, (kc > 0 || tap > 0 || k > 0) ? 1u : 0u);
            acc.mma(a_hi + ko, a_hi + a_half + ko, b_lo + ko, 1u);
            acc.mma(a_hi + ko, a_hi + a_half + ko, b_hi + ko, 1u);
          }
          wgmma_commit();
          if (kc == kchunks - 1 && tap == 8 && lane == 0) mbar_arrive(&order_bar[cw ^ 1]);
          wgmma_wait<1>();                    // the previous tap's MMAs have retired: release its weight slot, and
          if (prev >= 0) release_w(prev);     // after the first tap of a chunk the previous chunk's halo slot
          if (prev_a >= 0) {
            if (lane == 0) mbar_arrive(&aempty_bar[prev_a]);
            prev_a = -1;
          }
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        prev_a = astage;
        if (++astage == NA) { astage = 0; aphase ^= 1; }
      }
      wgmma_wait<0>();
      acc.fence_operands();
      release_w(prev);
      if (lane == 0) mbar_arrive(&aempty_bar[prev_a]);
      conv_epilogue_tile<BN>(a, acc, my_stg, img, h0, w0, nt * BN, nt, r, c, 8, bar);
    }
    } else {
    // ================= consumer warpgroup: main loop + epilogue =================
    const int m = threadIdx.x;              // accumulator row = pixel index inside the patch
    const int r = m >> a.tw_log2, c = m & (TW - 1);
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = worker; tile < a.total_tiles; tile += n_workers) {
      int img, h0, w0, nt;
      coords(tile, img, h0, w0, nt);
      Acc128<BN> acc;
      int prev = -1;
      for (int kit = 0; kit < kiters; ++kit) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = ring_a + stage * STAGE_BYTES;
        const uint64_t a_hi = gmma_desc_kmajor_sw128(sa), a_lo = gmma_desc_kmajor_sw128(sa + TC_A_BYTES);
        const uint64_t b_hi = gmma_desc_kmajor_sw128(sa + 2 * TC_A_BYTES);
        const uint64_t b_lo = gmma_desc_kmajor_sw128(sa + 2 * TC_A_BYTES + B_BYTES);
        constexpr uint64_t kHalf = (TC_BM / 2) * 128 / 16;   // pixel rows 64-127: +8 KiB
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) {
          // advance 16 bf16 = 32 bytes inside the 128-byte swizzle row: +2 in 16-byte units
          const uint64_t ko = (uint64_t)(k * 2);
          acc.mma(a_lo + ko, a_lo + kHalf + ko, b_hi + ko, (kit > 0 || k > 0) ? 1u : 0u);
          acc.mma(a_hi + ko, a_hi + kHalf + ko, b_lo + ko, 1u);
          acc.mma(a_hi + ko, a_hi + kHalf + ko, b_hi + ko, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();                      // the previous stage's MMAs have retired: release its slot
        if (prev >= 0) release_w(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      acc.fence_operands();
      if (prev >= 0) release_w(prev);
      conv_epilogue_tile<BN>(a, acc, stg, img, h0, w0, nt * BN, nt, r, c, TW);
    }
    }
  }
  __syncthreads();
}

// ---- host launcher --------------------------------------------------------------------------
template <int BN, int STAGES, bool HALO = false, int NA = 0, int WTW = 0>
static int launch_tc_variant(const CUtensorMap& xhi, const CUtensorMap& xlo, const CUtensorMap& whi,
                             const CUtensorMap& wlo, const ConvTcArgs& a, cudaStream_t s) {
  constexpr int smem = ConvTcSmem<BN, STAGES, HALO, NA, WTW>::BYTES;
  static_assert(smem <= 232448, "shared-memory budget");
  static DeviceOnce attr_done;   // the attribute is per device
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(conv3x3_tc_kernel<BN, STAGES, HALO, NA, WTW>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_done.mark();
  }
  const int sms = device_sm_count();
  const int grid = a.total_tiles < sms ? a.total_tiles : sms;
  conv3x3_tc_kernel<BN, STAGES, HALO, NA, WTW>
      <<<grid, ConvTcSmem<BN, STAGES, HALO, NA, WTW>::THREADS, smem, s>>>(xhi, xlo, whi, wlo, a);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

static int g_tc_bn_override = 0;   // test hook: force BN (64/128) of the 128-pixel kernels where it divides Cout
void tc_set_bn_override(int bn) { g_tc_bn_override = bn; }
static int g_tc_variant_override = 0;   // test hook: 1 forces the 128-pixel kernels, 2 the 256-pixel one
void tc_set_variant_override(int v) { g_tc_variant_override = v; }

int launch_conv3x3_tc(const __nv_bfloat16* x_hi, const __nv_bfloat16* x_lo, const ConvParams& p,
                      int N, int H, int W, int cin, int cout, bool relu, bool pool,
                      __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, float* y_f32, cudaStream_t s, float* ssq,
                      int* ssq_parts) {
  IBL_REQUIRE(cin % 64 == 0 && cout % 64 == 0, "tensor-core conv needs Cin%64==0 and Cout%64==0");
  IBL_REQUIRE(p.w_hi && p.w_lo, "tensor-core conv: weights were not re-laid-out");
  IBL_REQUIRE(H >= 1 && W >= 1 && N >= 1, "empty conv input");
  ConvTcArgs a{};
  a.N = N; a.H = H; a.W = W; a.cin = cin; a.cout = cout;
  // patch shape of the 128-pixel kernels: 8x16 or 16x8, whichever wastes fewer accumulator rows (pixels computed for
  // the map)
  auto waste = [&](int tw, int px) {
    int th = px / tw;
    return (long long)cdiv(W, tw) * tw * cdiv(H, th) * th;
  };
  const int tw128 = (waste(16, 128) <= waste(8, 128)) ? 16 : 8;
  // The 256-pixel kernel (64 output channels x 256 pixels per tile, weights in registers) on 16x16 patches wherever
  // they waste no more rows than the 128-pixel kernels: conv2_x and conv4_x at 480x640, not conv3_x at 120x160 (8x16
  // tiles it exactly, 16x16 wastes 6.7 %) or conv5_x at 30x40 (28 %).  The kernel's 8x32 patch tiles 120x160 exactly
  // but measured no faster there than the 128-pixel kernel (DESIGN 5, K1b), so it is not built.  Like the N tile below,
  // the choice depends on the layer's shape only, never on the batch, so an image's descriptor does not depend on the
  // batch it travels in (tests: bit-identical across batch compositions).
  constexpr int tw256 = 16;
  bool wide = waste(tw256, 256) <= waste(tw128, 128);
  if (g_tc_bn_override) wide = false;
  if (g_tc_variant_override) wide = g_tc_variant_override == 2;
  const int TW = wide ? tw256 : tw128, TH = (wide ? TC_WIDE_PX : TC_BM) / TW;
  a.tw_log2 = TW == 16 ? 4 : 3;
  a.tiles_w = cdiv(W, TW);
  a.tiles_h = cdiv(H, TH);
  // N tile of the 128-pixel kernels: 128 where Cout allows (the accumulator is 128 registers per consumer thread), 64
  // for Cout = 64; the 256-pixel kernel's tile is 64 channels.
  int bn = wide ? 64 : cout % 128 == 0 ? 128 : 64;
  if (!wide && g_tc_bn_override && cout % g_tc_bn_override == 0 && (g_tc_bn_override == 64 || g_tc_bn_override == 128))
    bn = g_tc_bn_override;
  // Halo staging on the 128-wide and the 256-pixel tiles.  The 128-pixel kernels walk K in different orders, so the
  // choice depends on Cout only; the patch shape only moves pixels between accumulator rows, not the order of any
  // pixel's sums.
  const bool halo = wide || bn == 128;
  a.n_tiles = cout / bn;
  a.total_tiles = (int)((long long)N * a.tiles_h * a.tiles_w * a.n_tiles);
  a.relu = relu; a.pool = pool;
  a.bias = p.bias; a.y_hi = y_hi; a.y_lo = y_lo; a.y_f32 = y_f32;
  a.ssq = pool ? nullptr : ssq;
  a.ssq_stride = (long long)N * H * W;
  if (ssq_parts) *ssq_parts = wide ? cout / 16 : a.n_tiles;   // the 256-pixel kernel writes one partial per warp

  CUtensorMap m_xhi, m_xlo, m_whi, m_wlo;
  {
    uint64_t dims[4] = {(uint64_t)cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t str[3] = {(uint64_t)cin * 2, (uint64_t)W * cin * 2, (uint64_t)H * W * cin * 2};
    uint32_t box[4] = {64, (uint32_t)(halo ? TW + 2 : TW), (uint32_t)(halo ? TH + 2 : TH), 1};
    IBL_RET(make_tmap(&m_xhi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x_hi, dims, str, box));
    IBL_RET(make_tmap(&m_xlo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x_lo, dims, str, box));
  }
  {
    uint64_t dims[3] = {(uint64_t)cin, (uint64_t)cout, 9};
    uint64_t str[2] = {(uint64_t)cin * 2, (uint64_t)cout * cin * 2};
    uint32_t box[3] = {64, (uint32_t)bn, 1};
    IBL_RET(make_tmap(&m_whi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, p.w_hi, dims, str, box));
    IBL_RET(make_tmap(&m_wlo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, p.w_lo, dims, str, box));
  }
  if (wide) return launch_tc_variant<64, 3, true, 2, 16>(m_xhi, m_xlo, m_whi, m_wlo, a, s);
  if (halo) return launch_tc_variant<128, 3, true, 2>(m_xhi, m_xlo, m_whi, m_wlo, a, s);
  return launch_tc_variant<64, 4>(m_xhi, m_xlo, m_whi, m_wlo, a, s);
}

// =====================================================================================================================
// conv1_1 + conv1_2 (+ ReLU + 2x2 max-pool) in ONE kernel  (vgg.py:40-42 slots 0 and 2)
//
// conv1_1's output -- 64 channels at full resolution, 2.5 GB per batch of 32 as hi/lo planes -- is the largest tensor
// of the network and would be written to HBM by one kernel only to be read back by the next.  Here a CTA owns 16 x 16
// patches of conv1_2 outputs and RECOMPUTES the conv1_1 activations each needs, the (16+2) x (16+2) = 324-pixel halo,
// straight into a shared-memory halo tile laid out as the wide tiles' (18-pixel rows, TC_WIDE_HALO_PLANE per plane).
//
//   producer (warpgroup 0)     warp 0: TMA ring of conv1_2's weight taps (16 KiB each); the warpgroup's registers go
//                              to the consumers (setmaxnreg)
//   consumers (warpgroups 1-2) consumer j takes the CTA's tiles j, j + 2, ... and, per tile:
//     A1  im2col of the 3-channel input for the 324 halo pixels: K = 27 -> 32, bf16 hi/lo, 64-byte K-major SW64 rows,
//         384 rows = 6 m64 tiles, built in the consumer's own halo buffer (f1_a1_off)
//     C1  conv1_1 per m64 tile: 2 K steps x 3 wgmma (N = 64) -> bias, ReLU, ZERO outside the image (conv1_2's padding),
//         hi/lo straight from the accumulator fragment into the halo tile's swizzled rows; two tiles in flight, so one
//         tile's MMAs run during the epilogue of the tile before.  (Two more tiles' accumulators, 128 registers, make
//         ptxas spill and serialise C2's register-A MMAs.)
//     C2  conv1_2 with the wide tiles' operand roles: M = the 64 output channels, A = the tap's weights in registers
//         (ldsm_a_sw128), N = the 256 pixels as two n128 views of the halo tile; 9 taps x 4 K steps x 2 views x 3 wgmma
//         -> 2x2 max-pool, bias, ReLU, hi/lo planes -> HBM, register-local                   [conv_wide_epilogue]
// so one consumer's C2 MMAs run while the other does its C2 epilogue, its next tile's A1, C1 and C1 epilogue.  Both
// convolutions add their products in the order of the unfused path (conv1_1_tc_kernel, then conv3x3_tc_kernel on
// conv1_2): lo.hi, hi.lo, hi.hi per k16 step into one accumulator.
// =====================================================================================================================
struct Conv1FusedArgs {
  const float* x;       // [N,3,H,W]
  const float* w1;      // conv1_1 OIHW [64,3,3,3]
  const float* bias1;   // [64]
  ConvTcArgs c2;        // conv1_2: N,H,W, cin = cout = 64, tw_log2 = 4, tiles, relu, pool, bias, y_hi / y_lo
};

constexpr int F1_HALO_W = 18;                             // halo row pitch (pixels) of a 16x16 patch
constexpr int F1_HALO_ROWS = F1_HALO_W * F1_HALO_W;       // 324
constexpr int F1_HALO_STAGE = 2 * TC_WIDE_HALO_PLANE;     // hi | lo
constexpr int F1_A1_TILE = 64 * 64;                      // one m64 tile of A1 per plane: 64-byte rows, K = 32
constexpr int F1_W1_PLANE = 64 * 64;                      // conv1_1 filters: 64 rows x 64 B per plane
constexpr int F1_W2_STAGE = 2 * 64 * TC_BK * 2;           // one tap of conv1_2: W_hi 8 KiB | W_lo 8 KiB
constexpr int F1_W2_STAGES = 3;
// [halo 0 | halo 1] [3 weight taps] [W1 hi | W1 lo] [barriers, bias1]
constexpr int F1_OFF_W2 = 2 * F1_HALO_STAGE;              // 164 KiB
constexpr int F1_OFF_W1 = F1_OFF_W2 + F1_W2_STAGES * F1_W2_STAGE;
constexpr int F1_OFF_BAR = F1_OFF_W1 + 2 * F1_W1_PLANE;
constexpr int F1_SMEM = F1_OFF_BAR + 512 + 1024;

// A1 plane `plane` (0 hi, 1 lo) of m64 tile g (rows 64 g .. 64 g + 63), as a byte offset into the consumer's halo
// buffer.  Tile g's C1 epilogue writes halo rows 64 g .. 64 g + 63 of both planes while tile g + 1's MMAs still read, so
// tiles 0-4 keep both A1 planes in their own rows of the hi halo plane.  Tile 5 (halo rows 320-323; the hi plane has no
// room for its 8 KiB there) goes first and keeps its A1 in the lo plane's rows 0-63, which tile 0's epilogue overwrites
// only after tile 5 has retired.
__host__ __device__ constexpr int f1_a1_off(int g, int plane) {
  return (g < 5 ? g * 2 * F1_A1_TILE : TC_WIDE_HALO_PLANE) + plane * F1_A1_TILE;
}
static_assert(2 * F1_A1_TILE == 64 * 128, "a tile's A1 fills its own halo rows of the hi plane");
static_assert(5 * 64 < F1_HALO_ROWS && 6 * 64 >= F1_HALO_ROWS && f1_a1_off(4, 1) + F1_A1_TILE <= TC_WIDE_HALO_PLANE &&
                  F1_HALO_ROWS * 128 <= TC_WIDE_HALO_PLANE,
              "six m64 tiles cover the halo, only tile 5 reaches past halo row 319, and the halo tile fits in a plane");
static_assert(F1_HALO_STAGE % 1024 == 0 && F1_OFF_W2 % 1024 == 0 && F1_OFF_W1 % 512 == 0 && f1_a1_off(5, 1) % 512 == 0,
              "swizzle atom alignment");
static_assert(F1_SMEM <= 232448, "shared-memory budget of the fused conv1 kernel");

__global__ void __launch_bounds__(384, 1)
conv1_fused_tc_kernel(const __grid_constant__ CUtensorMap tm_whi, const __grid_constant__ CUtensorMap tm_wlo,
                      const Conv1FusedArgs fa) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const ConvTcArgs& a = fa.c2;
  uint8_t* w1 = smem + F1_OFF_W1;
  uint8_t* w2 = smem + F1_OFF_W2;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + F1_OFF_BAR);
  uint64_t* w_full = bars;                           // [3] producer
  uint64_t* w_empty = bars + F1_W2_STAGES;           // [3] 4 warps of the consumer of the tile
  uint64_t* order_bar = bars + 2 * F1_W2_STAGES;     // [2] 4 warps of the other consumer
  float* bias1_s = reinterpret_cast<float*>(bars + 16);   // [64]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // one-time: conv1_1's filters as K-major SW64 rows, k = tap*3 + c (zero for k >= 27)
  for (int i = threadIdx.x; i < 64 * 4; i += blockDim.x) {   // (row n, 16-byte chunk j): 8 k-values each
    const int n = i >> 2, j = i & 3;
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float v[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int k = j * 8 + e * 2 + u;
        v[u] = 0.f;
        if (k < 27) v[u] = fa.w1[(n * 3 + (k % 3)) * 9 + (k / 3)];
      }
      const __nv_bfloat16 h0 = __float2bfloat16_rn(v[0]), h1 = __float2bfloat16_rn(v[1]);
      __nv_bfloat162 hh(h0, h1);
      hi[e] = *reinterpret_cast<uint32_t*>(&hh);
      lo[e] = pack_bf16x2(v[0] - __bfloat162float(h0), v[1] - __bfloat162float(h1));
    }
    const int pos = n * 64 + ((j ^ ((n >> 1) & 3)) * 16);
    *reinterpret_cast<uint4*>(w1 + pos) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(w1 + F1_W1_PLANE + pos) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
  if (threadIdx.x < 64) bias1_s[threadIdx.x] = fa.bias1[threadIdx.x];
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_whi);
    tma_prefetch_desc(&tm_wlo);
    for (int i = 0; i < F1_W2_STAGES; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 4); }
    mbar_init(&order_bar[0], 4);
    mbar_init(&order_bar[1], 4);
    fence_barrier_init();
  }
  fence_proxy_async();        // generic-proxy writes of the filters -> visible to the tensor core
  __syncthreads();
  const int tiles_per_img = a.tiles_h * a.tiles_w;
  auto coords = [&](int tile, int& img, int& h0, int& w0) {
    img = tile / tiles_per_img;
    const int rem = tile - img * tiles_per_img;
    h0 = (rem / a.tiles_w) * 16;
    w0 = (rem % a.tiles_w) * 16;
  };

  if (warp < 4) setmaxnreg_dec<40>();
  if (warp == 0) {
    // ================= TMA producer: conv1_2 weight taps (convergent warp, one elected lane issues) =================
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < a.total_tiles; tile += gridDim.x) {
      for (int tap = 0; tap < 9; ++tap) {
        mbar_wait_warp(&w_empty[stage], phase ^ 1);
        uint8_t* st = w2 + stage * F1_W2_STAGE;
        if (elect_one()) {
          mbar_arrive_expect_tx(&w_full[stage], F1_W2_STAGE);
          tma_load_3d(st, &tm_whi, &w_full[stage], 0, 0, tap);
          tma_load_3d(st + F1_W2_STAGE / 2, &tm_wlo, &w_full[stage], 0, 0, tap);
        }
        __syncwarp();
        if (++stage == F1_W2_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ================= two consumer warpgroups (ping-pong): A1 -> C1 -> halo tile, C2 -> conv1_2 epilogue =================
    setmaxnreg_inc<232>();
    const int cw = warp / 4 - 1;                      // consumer 0 / 1
    const int bar = 1 + cw;                           // its named barrier
    uint8_t* halo = smem + cw * F1_HALO_STAGE;        // this consumer's halo tile; A1 inside it until C1 retires
    const int t = threadIdx.x & 127;                  // thread inside the warpgroup
    const uint32_t ha = smem_u32(halo);
    const uint32_t w2a = smem_u32(w2);
    const uint64_t b1h = gmma_desc_kmajor_sw64(smem_u32(w1)), b1l = gmma_desc_kmajor_sw64(smem_u32(w1) + F1_W1_PLANE);
    constexpr uint64_t kA1Tile = 64 * 64 / 16;         // the next m64 tile of A1: +4 KiB
    // K-major SW128 view of the halo tile: 8-pixel groups one halo row (2304 B) apart; view v starts 8v pixels into
    // patch row 0 (+1 KiB)
    constexpr uint64_t kHaloDesc = ((uint64_t)1 << 16) | ((uint64_t)((F1_HALO_W * 128) >> 4) << 32) | ((uint64_t)1 << 62);
    // conv1_2's weight row map, as in the wide halo kernel: accumulator rows 16w + j and 16w + j + 8 (j < 8) read output
    // channels 16w + 2j + s and 16w + 2j + (s ^ 1), s = j >> 2, so a thread's two rows are adjacent channels
    const int wq = (threadIdx.x >> 5) & 3, jl = lane & 7, hl8 = (lane >> 3) & 1;
    const int wrow = 16 * wq + 2 * jl + (hl8 ^ (jl >> 2));
    const long long HW = (long long)a.H * a.W;
    // Consumer cw takes the CTA's tiles cw, cw + 2, ...  The producer fills the weight ring in tile order, so the taps of
    // CTA-local tile i start at running index 9 i.  The order barrier lets a consumer wait on its first tap only after
    // the other consumer has waited on all the taps of the tile before: a slot's full barrier is then at most one phase
    // behind the awaited one, so its parity is exact.
    for (int i = cw; blockIdx.x + i * gridDim.x < a.total_tiles; i += 2) {
      int img, h0, w0;
      coords(blockIdx.x + i * gridDim.x, img, h0, w0);
      // the per-row index math below is recomputed for every tile: hoisted out of the loop it would hold registers
      // through the C2 main loop and epilogue
      int tl = t;
      asm volatile("" : "+r"(tl));
      // ---- A1: rows t, t + 128, t + 256 (halo pixels; rows >= 324 are zero).  The epilogue has no barrier, so the
      // warpgroup meets here: every warp's previous C2 MMAs, the last readers of this buffer, have retired.
      wg_sync(bar);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int p = q * 128 + tl;
        float v[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) v[k] = 0.f;
        const int hl = p / F1_HALO_W, wl = p - hl * F1_HALO_W;
        const int ph = h0 - 1 + hl, pw = w0 - 1 + wl;
        if (p < F1_HALO_ROWS && ph >= 0 && ph < a.H && pw >= 0 && pw < a.W && img < a.N) {
          const float* xb = fa.x + (long long)img * 3 * HW;
#pragma unroll
          for (int tap = 0; tap < 9; ++tap) {
            const int ih = ph + tap / 3 - 1, iw = pw + tap % 3 - 1;
            if (ih >= 0 && ih < a.H && iw >= 0 && iw < a.W) {
              const long long o = (long long)ih * a.W + iw;
#pragma unroll
              for (int ci = 0; ci < 3; ++ci) v[tap * 3 + ci] = __ldg(xb + ci * HW + o);
            }
          }
        }
        const int g = p >> 6, r = p & 63;              // row r of m64 tile g
        uint8_t* rh = halo + f1_a1_off(g, 0) + r * 64;
        uint8_t* rl = halo + f1_a1_off(g, 1) + r * 64;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float x0 = v[8 * j + 2 * e], x1 = v[8 * j + 2 * e + 1];
            const __nv_bfloat16 h0b = __float2bfloat16_rn(x0), h1b = __float2bfloat16_rn(x1);
            __nv_bfloat162 hv(h0b, h1b);
            hi[e] = *reinterpret_cast<uint32_t*>(&hv);
            lo[e] = pack_bf16x2(x0 - __bfloat162float(h0b), x1 - __bfloat162float(h1b));
          }
          const int pos = (j ^ ((r >> 1) & 3)) * 16;
          *reinterpret_cast<uint4*>(rh + pos) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          *reinterpret_cast<uint4*>(rl + pos) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
      }
      fence_proxy_async();                             // generic-proxy writes of A1 -> visible to the tensor core
      wg_sync(bar);
      // ---- C1: conv1_1 on the six m64 tiles of A1 in the order 5, 0, 1, 2, 3, 4 (f1_a1_off), two in flight: step s
      // takes tile g from c1[s & 1] to halo rows 64 g .. 64 g + 63, then issues step s + 2's tile into c1[s & 1]
      float c1[2][32];
      auto issue_c1 = [&](int g, float (&acc)[32]) {
        const uint64_t a1h = gmma_desc_kmajor_sw64(ha + f1_a1_off(g, 0));
        const uint64_t a1l = gmma_desc_kmajor_sw64(ha + f1_a1_off(g, 1));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 2; ++k) {                  // K = 32: two 16-wide steps
          const uint64_t ko = (uint64_t)(k * 2);
          Wgmma<64, false, 0, 0>::mma(acc, a1l + ko, b1h + ko, k > 0 ? 1u : 0u);
          Wgmma<64, false, 0, 0>::mma(acc, a1h + ko, b1l + ko, 1u);
          Wgmma<64, false, 0, 0>::mma(acc, a1h + ko, b1h + ko, 1u);
        }
        wgmma_commit();
      };
      issue_c1(5, c1[0]);
      issue_c1(0, c1[1]);
#pragma unroll
      for (int step = 0; step < 6; ++step) {
        const int g = step == 0 ? 5 : step - 1;
        float (&acc)[32] = c1[step & 1];
        if (step < 5) wgmma_wait<1>(); else wgmma_wait<0>();   // the groups are committed in step order
#pragma unroll
        for (int j = 0; j < 32; ++j) asm volatile("" : "+f"(acc[j])::"memory");
        wg_sync(bar);                                  // no warp reads tile g's A1 any more: its halo rows may overwrite it
        // bias, ReLU, image mask, hi/lo -> halo row p, from the fragment.  Thread 32 w + l holds rows 16 w + l/4 (+ 8)
        // of the m64 tile, channel pairs 8 j + 2 (l % 4): one 4-byte store per plane and pair, eight distinct rows x
        // four lanes per 16-byte chunk position -> conflict-free.
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const int p = 64 * g + (tl & ~31) / 2 + ((tl & 31) >> 2) + 8 * hf;
          if (p < F1_HALO_ROWS) {
            const int hl = p / F1_HALO_W, wl = p - hl * F1_HALO_W;
            const int ph = h0 - 1 + hl, pw = w0 - 1 + wl;
            const bool inside = ph >= 0 && ph < a.H && pw >= 0 && pw < a.W && img < a.N;
            uint8_t* rh = halo + p * 128 + (tl & 3) * 4;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int ch = 8 * j + 2 * (tl & 3);
              float x0 = fmaxf(acc[4 * j + 2 * hf] + bias1_s[ch], 0.f);
              float x1 = fmaxf(acc[4 * j + 2 * hf + 1] + bias1_s[ch + 1], 0.f);
              if (!inside) { x0 = 0.f; x1 = 0.f; }       // conv1_2 pads its INPUT with zeros
              const __nv_bfloat16 h0b = __float2bfloat16_rn(x0), h1b = __float2bfloat16_rn(x1);
              __nv_bfloat162 hv(h0b, h1b);
              const int pos = (j ^ (p & 7)) * 16;
              *reinterpret_cast<uint32_t*>(rh + pos) = *reinterpret_cast<uint32_t*>(&hv);
              *reinterpret_cast<uint32_t*>(rh + TC_WIDE_HALO_PLANE + pos) =
                  pack_bf16x2(x0 - __bfloat162float(h0b), x1 - __bfloat162float(h1b));
            }
          }
        }
        if (step + 2 < 6) issue_c1(step + 1, acc);     // step s + 2 takes tile s + 1
      }
      fence_proxy_async();                             // generic-proxy writes of the halo -> visible to the tensor core
      wg_sync(bar);                                    // every halo row is written
      // ---- C2: conv1_2 over the nine tap views of the halo tile
      int stage = (i * 9) % F1_W2_STAGES;
      uint32_t phase = (uint32_t)((i * 9) / F1_W2_STAGES) & 1u;
      if (i > 0) mbar_wait(&order_bar[cw], (uint32_t)((i - 1) >> 1) & 1u);
      AccWide acc;
      // the weight fragments of one k16 step go into fw[k & 1] while the previous step's MMAs run
      uint32_t fw[2][2][4];
      int prev = -1;
#pragma unroll 1
      for (int tap = 0; tap < 9; ++tap) {
        mbar_wait(&w_full[stage], phase);
        const uint32_t sb = w2a + stage * F1_W2_STAGE;
        ldsm_a_sw128(fw[0][0], sb, wrow, 0);
        ldsm_a_sw128(fw[0][1], sb + F1_W2_STAGE / 2, wrow, 0);
        const uint32_t toff = (uint32_t)((tap / 3) * F1_HALO_W + tap % 3) * 128u;
        const uint64_t x_hi = kHaloDesc | (uint64_t)(((ha + toff) >> 4) & 0x3fffu);
        const uint64_t x_lo = kHaloDesc | (uint64_t)(((ha + TC_WIDE_HALO_PLANE + toff) >> 4) & 0x3fffu);
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) {
          const uint32_t(&fh)[4] = fw[k & 1][0];
          const uint32_t(&fl)[4] = fw[k & 1][1];
          const uint64_t ko = (uint64_t)(k * 2);
          wgmma_fence();
#pragma unroll
          for (int v = 0; v < 2; ++v) WgmmaRS<128>::mma(acc.d[v], fh, x_lo + 64 * v + ko, (tap > 0 || k > 0) ? 1u : 0u);
#pragma unroll
          for (int v = 0; v < 2; ++v) WgmmaRS<128>::mma(acc.d[v], fl, x_hi + 64 * v + ko, 1u);
#pragma unroll
          for (int v = 0; v < 2; ++v) WgmmaRS<128>::mma(acc.d[v], fh, x_hi + 64 * v + ko, 1u);
          wgmma_commit();
          if (k == 3 && tap == 8 && lane == 0) mbar_arrive(&order_bar[cw ^ 1]);
          wgmma_wait<1>();                             // the previous k16 step's MMAs have retired: its fragments are
          if (k == 0 && prev >= 0 && lane == 0) mbar_arrive(&w_empty[prev]);   // free, after k = 0 the previous tap's slot
          if (k + 1 < TC_BK / 16) {
            ldsm_a_sw128(fw[(k + 1) & 1][0], sb, wrow, k + 1);
            ldsm_a_sw128(fw[(k + 1) & 1][1], sb + F1_W2_STAGE / 2, wrow, k + 1);
          }
        }
        prev = stage;
        if (++stage == F1_W2_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int v = 0; v < 2; ++v)
#pragma unroll
        for (int e = 0; e < 64; ++e) asm volatile("" : "+f"(acc.d[v][e])::"memory");
      if (lane == 0) mbar_arrive(&w_empty[prev]);
      conv_wide_epilogue(a, acc, img, h0, w0, 0);
    }
  }
  __syncthreads();
}

// x [N,3,H,W] fp32 -> conv1_1 -> ReLU -> conv1_2 -> ReLU -> 2x2 max-pool as hi/lo planes [N,H/2,W/2,64]
int launch_conv1_fused_tc(const float* x_nchw, const float* w1_oihw, const float* bias1, const ConvParams& p2, int N, int H,
                          int W, __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, cudaStream_t s) {
  IBL_REQUIRE(p2.w_hi && p2.w_lo && p2.bias, "fused conv1: conv1_2 weights were not re-laid-out");
  Conv1FusedArgs fa{};
  fa.x = x_nchw; fa.w1 = w1_oihw; fa.bias1 = bias1;
  ConvTcArgs& a = fa.c2;
  a.N = N; a.H = H; a.W = W; a.cin = 64; a.cout = 64;
  a.tw_log2 = 4;
  a.tiles_w = cdiv(W, 16);
  a.tiles_h = cdiv(H, 16);
  a.n_tiles = 1;
  a.total_tiles = (int)((long long)N * a.tiles_h * a.tiles_w);
  a.relu = 1; a.pool = 1;
  a.bias = p2.bias; a.y_hi = y_hi; a.y_lo = y_lo; a.y_f32 = nullptr; a.ssq = nullptr; a.ssq_stride = 0;
  CUtensorMap m_whi, m_wlo;
  {
    uint64_t dims[3] = {64, 64, 9};
    uint64_t str[2] = {64 * 2, 64 * 64 * 2};
    uint32_t box[3] = {64, 64, 1};
    IBL_RET(make_tmap(&m_whi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, p2.w_hi, dims, str, box));
    IBL_RET(make_tmap(&m_wlo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, p2.w_lo, dims, str, box));
  }
  static DeviceOnce attr_done;   // the attribute is per device
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(conv1_fused_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, F1_SMEM));
    attr_done.mark();
  }
  const int sms = device_sm_count();
  const int grid = a.total_tiles < sms ? a.total_tiles : sms;
  conv1_fused_tc_kernel<<<grid, 384, F1_SMEM, s>>>(m_whi, m_wlo, fa);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ---- 2x2 max-pool on hi/lo planes (used only when the conv epilogue did not pool) -------------
__global__ void maxpool2x2_planes_kernel(const __nv_bfloat16* __restrict__ hi,
                                         const __nv_bfloat16* __restrict__ lo, int N, int H, int W,
                                         int C, __nv_bfloat16* __restrict__ yhi,
                                         __nv_bfloat16* __restrict__ ylo) {
  const int OH = H / 2, OW = W / 2;
  const long long total = (long long)N * OH * OW * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int ow = (int)(r % OW);
    r /= OW;
    const int oh = (int)(r % OH);
    const long long n = r / OH;
    float best = -INFINITY;
    __nv_bfloat16 bh = __float2bfloat16_rn(0.f), bl = bh;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const long long src = ((n * H + oh * 2 + dy) * (long long)W + ow * 2 + dx) * C + c;
        const __nv_bfloat16 a = hi[src], b = lo[src];
        const float v = __bfloat162float(a) + __bfloat162float(b);
        if (v > best) { best = v; bh = a; bl = b; }
      }
    yhi[i] = bh;
    ylo[i] = bl;
  }
}

int launch_maxpool2x2_planes(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int N, int H, int W,
                             int C, __nv_bfloat16* yhi, __nv_bfloat16* ylo, cudaStream_t s) {
  long long total = (long long)N * (H / 2) * (W / 2) * C;
  unsigned blocks = (unsigned)((total + 255) / 256);
  if (blocks > 132 * 32) blocks = 132 * 32;
  if (!blocks) blocks = 1;
  maxpool2x2_planes_kernel<<<blocks, 256, 0, s>>>(hi, lo, N, H, W, C, yhi, ylo);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

int tc_selftest(float* max_rel_err, cudaStream_t s) {
  (void)s;
  if (max_rel_err) *max_rel_err = 0.f;
  return tc_driver_init();
}

}  // namespace ibl
