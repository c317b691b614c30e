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
// Warp roles (160 threads, persistent over tiles):
//   warps 0-3  consumer warpgroup: wgmma main loop (two m64 halves of the 128-pixel tile), then the epilogue
//   warp 4     TMA producer
// Epilogue: accumulator -> row-per-thread views (Acc128::rows32), + bias, ReLU, optional fused 2x2 max-pool
// (warp shuffles), split into hi/lo planes (or fp32 for conv5_3), 16-byte stores.
#include <stdlib.h>

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
  int tw_log2;            // TW = 1 << tw_log2 (8 or 16), TH = 128 / TW
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
  float acc_scale;        // optional accumulator compensation factor (see tc_acc_scale)
};

// Optional compensation of a tensor-core accumulator that rounds toward zero: the epilogue multiplies the accumulator
// by 1 + n_mma * c (n_mma = k16 MMA steps accumulated into the tile) before the bias is added.  IBL_TC_BIAS_COMP=<c>
// sets c (default 0: the sm_90 accumulator needs no compensation at the 1e-4 descriptor tolerance).
static float tc_acc_scale(int cin) {
  static const float c = [] { const char* v = getenv("IBL_TC_BIAS_COMP"); return v ? (float)atof(v) : 0.f; }();
  return 1.f + (float)(27 * (cin / 16)) * c;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// One accumulator tile (128 pixel rows x BN output channels, thread = pixel row) to global memory:
// bias + ReLU + fused 2x2 max-pool + bf16 hi/lo split (or fp32), optional per-pixel sum of squares.
template <int BN>
__device__ __forceinline__ void conv_epilogue_tile(const ConvTcArgs& a, const Acc128<BN>& acc, float* stg, int img, int h0,
                                                   int w0, int n0, int nt, int r, int c, int TW) {
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
    acc.rows32(ch, stg, raw);
    if (a.pool) {
      // 2x2 max-pool BEFORE bias / ReLU / split (fmaf(., scale > 0, b) and max(., 0) are monotone, so the results are
      // the same bits) as a two-step exchange: against the w-neighbour (lane ^ 1) every lane keeps one half of the 32
      // channels and sends the other, against the h-neighbour (lane ^ TW) one half of those 16 -- 24 shuffles instead
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
        const float got = __shfl_xor_sync(0xffffffffu, s2 ? u[j] : u[j + 8], TW);
        w8[j] = fmaxf(s2 ? u[j + 8] : u[j], got);
      }
      if (valid) {
        const int cbase = n0 + ch * 32 + (s1 ? 16 : 0) + (s2 ? 8 : 0);
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(a.bias + cbase));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(a.bias + cbase) + 1);
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          w8[j] = fmaf(w8[j], a.acc_scale, bb[j]);
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
      v[4 * j + 0] = fmaf(__uint_as_float(raw[4 * j + 0]), a.acc_scale, b.x);
      v[4 * j + 1] = fmaf(__uint_as_float(raw[4 * j + 1]), a.acc_scale, b.y);
      v[4 * j + 2] = fmaf(__uint_as_float(raw[4 * j + 2]), a.acc_scale, b.z);
      v[4 * j + 3] = fmaf(__uint_as_float(raw[4 * j + 3]), a.acc_scale, b.w);
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
// TMA-written tile correctly (pinned on hardware by tests/test_gpu_variants.py through tc_probe.cu).
// L2->SM traffic of the A operand drops from 9 x 32 KiB to 45 KiB per chunk; the weights get their own ring.
constexpr int TC_HALO_W = 10, TC_HALO_H = 18;
constexpr int TC_HALO_PLANE = 23 * 1024;        // 180 rows x 128 B = 23040 B, padded to the swizzle period
constexpr int TC_HALO_STAGE = 2 * TC_HALO_PLANE;

template <int BN, int STAGES, bool HALO = false, int NA = 0>
struct ConvTcSmem {
  static constexpr int B_BYTES = BN * TC_BK * 2;
  static constexpr int STAGE_BYTES = HALO ? 2 * B_BYTES : 2 * TC_A_BYTES + 2 * B_BYTES;
  static constexpr int A_RING = HALO ? NA * TC_HALO_STAGE : 0;
  static constexpr int BYTES = A_RING + STAGES * STAGE_BYTES + ACC_STG_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

// PAIR: the grid is launched as clusters of two CTAs ("SM pairs") that share one work item = (two adjacent patches, one
// N tile).  Each CTA stages its own activations and fetches only HALF of every weight tap, TMA-multicasting it into both
// CTAs' shared memory: the per-SM L2->SM weight traffic halves.  A weight slot may be refilled only when the consumers
// of BOTH CTAs have released it (arrival count 8: every consumer warp arrives on both CTAs' barriers).
template <int BN, int STAGES, bool HALO, int NA, bool PAIR>
__global__ void __launch_bounds__(160, 1)
conv3x3_tc_kernel(const __grid_constant__ CUtensorMap tm_xhi, const __grid_constant__ CUtensorMap tm_xlo,
                  const __grid_constant__ CUtensorMap tm_whi, const __grid_constant__ CUtensorMap tm_wlo,
                  const ConvTcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle; dynamic smem base is only 16B-aligned
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  using L = ConvTcSmem<BN, STAGES, HALO, NA>;
  constexpr int B_BYTES = L::B_BYTES;
  constexpr int STAGE_BYTES = L::STAGE_BYTES;
  constexpr int A_RING = L::A_RING;           // HALO: the halo ring sits in front of the weight ring
  uint8_t* ring = smem + A_RING;
  float* stg = reinterpret_cast<float*>(ring + STAGES * STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + STAGES * STAGE_BYTES + ACC_STG_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* afull_bar = bars + 2 * STAGES;    // HALO only: [NA] + [NA]
  uint64_t* aempty_bar = afull_bar + NA;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
  const int worker = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
  const int n_workers = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tm_xhi);
    tma_prefetch_desc(&tm_xlo);
    tma_prefetch_desc(&tm_whi);
    tma_prefetch_desc(&tm_wlo);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], PAIR ? 8 : 4);   // one arrival per consumer warp (of both CTAs of a pair)
    }
    for (int i = 0; i < NA; ++i) {
      mbar_init(&afull_bar[i], 1);
      mbar_init(&aempty_bar[i], 4);
    }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();
  if (PAIR) cluster_sync_all();     // the peer's barriers exist before anything is multicast into this CTA

  const int TW = 1 << a.tw_log2;
  const int kchunks = a.cin / TC_BK;
  const int kiters = 9 * kchunks;
  const int tiles_per_img = a.tiles_h * a.tiles_w;
  auto coords = [&](int tile, int& img, int& h0, int& w0, int& nt) {
    nt = tile % a.n_tiles;
    // pair: an odd patch count leaves img == N for the last peer: TMA zero-fills, the epilogue stores nothing
    const int pt = PAIR ? 2 * (tile / a.n_tiles) + (int)rank : tile / a.n_tiles;
    img = pt / tiles_per_img;
    const int rem = pt - img * tiles_per_img;
    h0 = (rem / a.tiles_w) * (TC_BM >> a.tw_log2);
    w0 = (rem % a.tiles_w) * TW;
  };

  if (warp == 4) {
    // ================= TMA producer: convergent warp, one elected lane issues, coordinates warp-uniform =================
    const uint32_t smem_a = warp_uniform(smem_u32(smem));
    const uint32_t ring_a = smem_a + A_RING;
    const uint32_t bars_a = ring_a + STAGES * STAGE_BYTES + ACC_STG_BYTES;
    const uint32_t full_a = bars_a, empty_a = bars_a + 8 * STAGES;
    const uint32_t afull_a = bars_a + 16 * STAGES, aempty_a = afull_a + 8 * NA;
    const int rank_u = (int)warp_uniform(rank);
    // the two weight planes of one tap (into `st`, planes B_BYTES apart); a pair's CTAs each fetch one half of the rows
    auto load_w = [&](uint32_t st, uint32_t fb, int c0, int n0, int tap) {
      if (PAIR) {
        constexpr int HB = B_BYTES / 2;
        tma_load_3d_mc_a(st + rank_u * HB, &tm_whi, fb, c0, n0 + rank_u * (BN / 2), tap, 0x3);
        tma_load_3d_mc_a(st + B_BYTES + rank_u * HB, &tm_wlo, fb, c0, n0 + rank_u * (BN / 2), tap, 0x3);
      } else {
        tma_load_3d_a(st, &tm_whi, fb, c0, n0, tap);
        tma_load_3d_a(st + B_BYTES, &tm_wlo, fb, c0, n0, tap);
      }
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
          const uint32_t sa = smem_a + as_u * TC_HALO_STAGE;
          constexpr uint32_t kHaloBytes = 2u * TC_HALO_W * TC_HALO_H * 128u;
          if (elect_one()) {
            mbar_arrive_expect_tx_a(afull_a + 8 * as_u, kHaloBytes);
            tma_load_4d_a(sa, &tm_xhi, afull_a + 8 * as_u, c0, w0 - 1, h0 - 1, img);
            tma_load_4d_a(sa + TC_HALO_PLANE, &tm_xlo, afull_a + 8 * as_u, c0, w0 - 1, h0 - 1, img);
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
  } else {
    // ================= consumer warpgroup: main loop + epilogue =================
    const int m = threadIdx.x;              // accumulator row = pixel index inside the patch
    const int r = m >> a.tw_log2, c = m & (TW - 1);
    const uint32_t smem_a = smem_u32(smem);
    const uint32_t ring_a = smem_a + A_RING;
    int stage = 0, astage = 0;
    uint32_t phase = 0, aphase = 0;
    (void)ring_a; (void)astage; (void)aphase;
    auto release_w = [&](int st) {          // this warp is done reading weight slot st (in both CTAs' rings of a pair)
      if (lane == 0) {
        mbar_arrive(&empty_bar[st]);
        if (PAIR) mbar_arrive_remote(mapa_u32(smem_u32(&empty_bar[st]), rank ^ 1u));
      }
    };
    for (int tile = worker; tile < a.total_tiles; tile += n_workers) {
      int img, h0, w0, nt;
      coords(tile, img, h0, w0, nt);
      Acc128<BN> acc;
      int prev = -1;
      if constexpr (HALO) {
        // K-major SW128 view of the halo tile: 8-pixel row groups 10 rows apart; pixel rows 64-127 = groups 8-15
        constexpr uint64_t kHaloDesc = ((uint64_t)1 << 16) | ((uint64_t)((TC_HALO_W * 128) >> 4) << 32) | ((uint64_t)1 << 62);
        constexpr uint64_t kHalf = 8 * TC_HALO_W * 128 / 16;
        for (int kc = 0; kc < kchunks; ++kc) {
          mbar_wait(&afull_bar[astage], aphase);
          const uint32_t ha = smem_a + astage * TC_HALO_STAGE;
          for (int tap = 0; tap < 9; ++tap) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t toff = (uint32_t)((tap / 3) * TC_HALO_W + tap % 3) * 128u;
            const uint64_t a_hi = kHaloDesc | (uint64_t)(((ha + toff) >> 4) & 0x3fffu);
            const uint64_t a_lo = kHaloDesc | (uint64_t)(((ha + TC_HALO_PLANE + toff) >> 4) & 0x3fffu);
            const uint32_t sb = ring_a + stage * STAGE_BYTES;
            const uint64_t b_hi = gmma_desc_kmajor_sw128(sb), b_lo = gmma_desc_kmajor_sw128(sb + B_BYTES);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < TC_BK / 16; ++k) {
              const uint64_t ko = (uint64_t)(k * 2);
              acc.mma(a_lo + ko, a_lo + kHalf + ko, b_hi + ko, (kc > 0 || tap > 0 || k > 0) ? 1u : 0u);
              acc.mma(a_hi + ko, a_hi + kHalf + ko, b_lo + ko, 1u);
              acc.mma(a_hi + ko, a_hi + kHalf + ko, b_hi + ko, 1u);
            }
            wgmma_commit();
            if (tap < 8) {
              wgmma_wait<1>();
              if (prev >= 0) release_w(prev);
              prev = stage;
            } else {                              // the halo slot is free once all nine taps have retired
              wgmma_wait<0>();
              if (prev >= 0) release_w(prev);
              release_w(stage);
              if (lane == 0) mbar_arrive(&aempty_bar[astage]);
              prev = -1;
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
          if (++astage == NA) { astage = 0; aphase ^= 1; }
        }
      } else
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
  __syncthreads();
  if (PAIR) cluster_sync_all();     // no CTA leaves while its peer may still multicast into it or arrive on its barriers
}

// ---- host launcher --------------------------------------------------------------------------
template <int BN, int STAGES, bool HALO = false, int NA = 0>
static int launch_tc_variant(const CUtensorMap& xhi, const CUtensorMap& xlo, const CUtensorMap& whi,
                             const CUtensorMap& wlo, const ConvTcArgs& a, bool pair, cudaStream_t s) {
  constexpr int smem = ConvTcSmem<BN, STAGES, HALO, NA>::BYTES;
  static_assert(smem <= 232448, "shared-memory budget");
  static DeviceOnce attr_done;   // the attributes are per device
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(conv3x3_tc_kernel<BN, STAGES, HALO, NA, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    IBL_CUDA_OK(cudaFuncSetAttribute(conv3x3_tc_kernel<BN, STAGES, HALO, NA, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_done.mark();
  }
  const int sms = device_sm_count();
  if (!pair) {
    const int grid = a.total_tiles < sms ? a.total_tiles : sms;
    conv3x3_tc_kernel<BN, STAGES, HALO, NA, false><<<grid, 160, smem, s>>>(xhi, xlo, whi, wlo, a);
    IBL_CUDA_OK(cudaGetLastError());
    return IBL_OK;
  }
  // a.total_tiles counts pair work items; one 2-CTA cluster per item, at most sms/2 clusters
  const int pairs = a.total_tiles < sms / 2 ? a.total_tiles : sms / 2;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(2 * pairs);
  cfg.blockDim = dim3(160);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  IBL_CUDA_OK(cudaLaunchKernelEx(&cfg, conv3x3_tc_kernel<BN, STAGES, HALO, NA, true>, xhi, xlo, whi, wlo, a));
  return IBL_OK;
}

static int g_tc_bn_override = 0;   // test hook: force BN (64/128) where it divides Cout
void tc_set_bn_override(int bn) { g_tc_bn_override = bn; }

int launch_conv3x3_tc(const __nv_bfloat16* x_hi, const __nv_bfloat16* x_lo, const ConvParams& p,
                      int N, int H, int W, int cin, int cout, bool relu, bool pool,
                      __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, float* y_f32, cudaStream_t s, float* ssq,
                      int* ssq_parts) {
  IBL_REQUIRE(cin % 64 == 0 && cout % 64 == 0, "tensor-core conv needs Cin%64==0 and Cout%64==0");
  IBL_REQUIRE(p.w_hi && p.w_lo, "tensor-core conv: weights were not re-laid-out");
  IBL_REQUIRE(H >= 1 && W >= 1 && N >= 1, "empty conv input");
  ConvTcArgs a{};
  a.N = N; a.H = H; a.W = W; a.cin = cin; a.cout = cout;
  // patch shape: 8x16 or 16x8, whichever wastes fewer accumulator rows
  auto waste = [&](int tw) {
    int th = 128 / tw;
    return (long long)cdiv(W, tw) * tw * cdiv(H, th) * th;
  };
  a.tw_log2 = (waste(16) <= waste(8)) ? 4 : 3;
  const int TW = 1 << a.tw_log2, TH = 128 / TW;
  a.tiles_w = cdiv(W, TW);
  a.tiles_h = cdiv(H, TH);
  // N tile: 128 where Cout allows (the accumulator is 128 registers per consumer thread), 64 for Cout = 64.  The
  // choice depends on Cout only, never on the batch, so an image's descriptor does not depend on the batch it
  // travels in (tests: bit-identical across batch compositions).
  int bn = cout % 128 == 0 ? 128 : 64;
  if (g_tc_bn_override && cout % g_tc_bn_override == 0 && (g_tc_bn_override == 64 || g_tc_bn_override == 128))
    bn = g_tc_bn_override;
  // Halo staging (16x8 patches): IBL_CONV_HALO=0 never, =1 (default) on the 128-wide tiles, =2 on every N tile.  The
  // choice depends on Cout only, never on the batch (the variants walk K in different orders).
  static const int halo_env = [] { const char* v = getenv("IBL_CONV_HALO"); return v ? atoi(v) : 1; }();
  const bool halo = halo_env == 2 || (halo_env == 1 && bn == 128);
  if (halo) {
    a.tw_log2 = 3;
    a.tiles_w = cdiv(W, 8);
    a.tiles_h = cdiv(H, 16);
  }
  // SM pairs (weight taps multicast to two CTAs with adjacent patches): IBL_CONV_2SM=0 (default) never, =1 where the
  // weights are the larger operand stream (Cin >= 256: conv3_2 .. conv5_3), =2 on every layer.  Measured on an H100 at
  // batch 32 x 480x640: =1 gave 949 images/s against 1063 without pairs (the cluster-wide slot release costs more
  // than the halved weight traffic saves), hence off by default.  Each CTA still computes its own patch in the same
  // order, so the results do not depend on the choice.
  static const int pair_env = [] { const char* v = getenv("IBL_CONV_2SM"); return v ? atoi(v) : 0; }();
  const long long patches = (long long)N * a.tiles_h * a.tiles_w;
  const bool pair = patches >= 2 && (pair_env == 2 || (pair_env == 1 && cin >= 256));
  a.n_tiles = cout / bn;
  a.total_tiles = (int)((pair ? (patches + 1) / 2 : patches) * a.n_tiles);
  a.relu = relu; a.pool = pool;
  a.bias = p.bias; a.y_hi = y_hi; a.y_lo = y_lo; a.y_f32 = y_f32;
  a.ssq = pool ? nullptr : ssq;
  a.ssq_stride = (long long)N * H * W;
  a.acc_scale = tc_acc_scale(cin);
  if (ssq_parts) *ssq_parts = a.n_tiles;

  CUtensorMap m_xhi, m_xlo, m_whi, m_wlo;
  {
    uint64_t dims[4] = {(uint64_t)cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t str[3] = {(uint64_t)cin * 2, (uint64_t)W * cin * 2, (uint64_t)H * W * cin * 2};
    uint32_t box[4] = {64, (uint32_t)(halo ? TC_HALO_W : TW), (uint32_t)(halo ? TC_HALO_H : TH), 1};
    IBL_RET(make_tmap(&m_xhi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x_hi, dims, str, box));
    IBL_RET(make_tmap(&m_xlo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x_lo, dims, str, box));
  }
  {
    uint64_t dims[3] = {(uint64_t)cin, (uint64_t)cout, 9};
    uint64_t str[2] = {(uint64_t)cin * 2, (uint64_t)cout * cin * 2};
    uint32_t box[3] = {64, (uint32_t)(pair ? bn / 2 : bn), 1};
    IBL_RET(make_tmap(&m_whi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, p.w_hi, dims, str, box));
    IBL_RET(make_tmap(&m_wlo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, p.w_lo, dims, str, box));
  }
  if (halo) {
    if (bn == 64) return launch_tc_variant<64, 4, true, 3>(m_xhi, m_xlo, m_whi, m_wlo, a, pair, s);
    return launch_tc_variant<128, 3, true, 2>(m_xhi, m_xlo, m_whi, m_wlo, a, pair, s);
  }
  if (bn == 64) return launch_tc_variant<64, 4>(m_xhi, m_xlo, m_whi, m_wlo, a, pair, s);
  return launch_tc_variant<128, 3>(m_xhi, m_xlo, m_whi, m_wlo, a, pair, s);
}

// =====================================================================================================================
// conv1_1 + conv1_2 (+ ReLU + 2x2 max-pool) in ONE kernel  (vgg.py:40-42 slots 0 and 2)
//
// conv1_1's output -- 64 channels at full resolution, 2.5 GB per batch of 32 as hi/lo planes -- is the largest tensor
// of the network and would be written to HBM by one kernel only to be read back by the next.  Here a CTA owns a 16 x 8
// patch of conv1_2 outputs and RECOMPUTES the conv1_1 activations it needs, the (16+2) x (8+2) = 180-pixel halo,
// straight into the shared-memory halo tile that conv1_2's nine tap views read (the HALO staging above):
//
//   builders (warps 5-8)   im2col of the 3-channel input for the 180 halo pixels: K = 27 -> 32, bf16 hi/lo, K-major
//                          SW128 rows (two 128-row M tiles)                                    [as conv1_1_tc_kernel]
//   consumer (warps 0-3)   C1: 2 M tiles x 2 K steps x 3 wgmma (N = 64) -> bias, ReLU, ZERO outside the image
//                          (conv1_2's padding), hi/lo -> halo tile;  C2: 9 taps x 4 K steps x 3 wgmma -> bias, ReLU,
//                          2x2 max-pool, hi/lo planes -> HBM                                   [conv_epilogue_tile]
//   producer (warp 4)      TMA ring of conv1_2's weight taps (16 KiB each)
// The builders fill the operand of the next tile while the consumer runs C1/C2 of the current one.
// =====================================================================================================================
struct Conv1FusedArgs {
  const float* x;       // [N,3,H,W]
  const float* w1;      // conv1_1 OIHW [64,3,3,3]
  const float* bias1;   // [64]
  ConvTcArgs c2;        // conv1_2: N,H,W, cin = cout = 64, tw_log2 = 3, tiles, relu, pool, bias, y_hi / y_lo
};

constexpr int F1_W1 = 16384;                         // conv1_1 filters: hi 8 KiB | lo 8 KiB
constexpr int F1_A1_PLANE = 256 * 128;               // 256 halo rows x 128 B (K = 32 uses the first 64 B of a row)
constexpr int F1_A1 = 2 * F1_A1_PLANE;               // hi | lo
constexpr int F1_W2_STAGE = 2 * 64 * TC_BK * 2;      // one tap of conv1_2: W_hi 8 KiB | W_lo 8 KiB
constexpr int F1_W2_STAGES = 3;
constexpr int F1_OFF_A1 = F1_W1;
constexpr int F1_OFF_HALO = F1_OFF_A1 + F1_A1;       // 80 KiB, 1024-aligned
constexpr int F1_OFF_W2 = F1_OFF_HALO + TC_HALO_STAGE;
constexpr int F1_OFF_STG = F1_OFF_W2 + F1_W2_STAGES * F1_W2_STAGE;
constexpr int F1_OFF_BAR = F1_OFF_STG + ACC_STG_BYTES;
constexpr int F1_SMEM = F1_OFF_BAR + 512 + 1024;
static_assert(F1_SMEM <= 232448, "shared-memory budget of the fused conv1 kernel");

__global__ void __launch_bounds__(288, 1)
conv1_fused_tc_kernel(const __grid_constant__ CUtensorMap tm_whi, const __grid_constant__ CUtensorMap tm_wlo,
                      const Conv1FusedArgs fa) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const ConvTcArgs& a = fa.c2;
  uint8_t* w1_hi = smem;
  uint8_t* w1_lo = smem + 8192;
  uint8_t* a1 = smem + F1_OFF_A1;
  uint8_t* halo = smem + F1_OFF_HALO;
  uint8_t* w2 = smem + F1_OFF_W2;
  float* stg = reinterpret_cast<float*>(smem + F1_OFF_STG);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + F1_OFF_BAR);
  uint64_t* w_full = bars;                 // [3] producer
  uint64_t* w_empty = bars + 3;            // [3] 4 consumer warps
  uint64_t* a1_full = bars + 6;            // 4 builder warps
  uint64_t* a1_empty = bars + 7;           // 4 consumer warps
  float* bias1_s = reinterpret_cast<float*>(bars + 8);   // [64]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // one-time: zero A1 (the K >= 32 half of every row stays zero), lay out conv1_1's filters
  for (int i = threadIdx.x; i < F1_A1 / 16; i += blockDim.x) reinterpret_cast<uint4*>(a1)[i] = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < 64 * 8; i += blockDim.x) {   // (row n, chunk j): 8 k-values each, k = tap*3 + c
    const int n = i >> 3, j = i & 7;
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
    const int pos = n * 128 + ((j ^ (n & 7)) * 16);
    *reinterpret_cast<uint4*>(w1_hi + pos) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(w1_lo + pos) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
  if (threadIdx.x < 64) bias1_s[threadIdx.x] = fa.bias1[threadIdx.x];
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_whi);
    tma_prefetch_desc(&tm_wlo);
    for (int i = 0; i < F1_W2_STAGES; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 4); }
    mbar_init(a1_full, 4);
    mbar_init(a1_empty, 4);
    fence_barrier_init();
  }
  fence_proxy_async();        // generic-proxy writes of the filters and the zero fill -> visible to the tensor core
  __syncthreads();
  const int tiles_per_img = a.tiles_h * a.tiles_w;
  auto coords = [&](int tile, int& img, int& h0, int& w0) {
    img = tile / tiles_per_img;
    const int rem = tile - img * tiles_per_img;
    h0 = (rem / a.tiles_w) * 16;
    w0 = (rem % a.tiles_w) * 8;
  };
  const long long HW = (long long)a.H * a.W;

  if (warp == 4) {
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
  } else if (warp < 4) {
    // ================= consumer warpgroup: C1 -> halo tile, C2 -> conv1_2 epilogue =================
    const int t = threadIdx.x;
    const int r = t >> 3, c = t & 7;                  // 8-wide, 16-tall patch
    const uint64_t b1h = gmma_desc_kmajor_sw128(smem_u32(w1_hi)), b1l = gmma_desc_kmajor_sw128(smem_u32(w1_lo));
    constexpr uint64_t kHaloDesc = ((uint64_t)1 << 16) | ((uint64_t)((TC_HALO_W * 128) >> 4) << 32) | ((uint64_t)1 << 62);
    constexpr uint64_t kHaloHalf = 8 * TC_HALO_W * 128 / 16;   // pixel rows 64-127 of a tap view: groups 8-15
    const uint32_t ha = smem_u32(halo);
    int stage = 0; uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < a.total_tiles; tile += gridDim.x, ++it) {
      int img, h0, w0;
      coords(tile, img, h0, w0);
      mbar_wait(a1_full, it & 1);
#pragma unroll 1
      for (int mt = 0; mt < 2; ++mt) {
        const uint32_t sa = smem_u32(a1) + mt * 16384;
        const uint64_t ah = gmma_desc_kmajor_sw128(sa), al = gmma_desc_kmajor_sw128(sa + F1_A1_PLANE);
        constexpr uint64_t kHalf = 64 * 128 / 16;
        Acc128<64> c1;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 2; ++k) {                   // K = 32: two 16-wide steps
          const uint64_t ko = (uint64_t)(k * 2);
          c1.mma(al + ko, al + kHalf + ko, b1h + ko, k > 0 ? 1u : 0u);
          c1.mma(ah + ko, ah + kHalf + ko, b1l + ko, 1u);
          c1.mma(ah + ko, ah + kHalf + ko, b1h + ko, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        c1.fence_operands();
        if (mt == 1 && lane == 0) mbar_arrive(a1_empty);   // the builders may refill A1
        // epilogue 1: bias, ReLU, image mask, hi/lo -> halo row p (the previous tile's C2 has retired)
        const int p = mt * 128 + t;
        const int hl = p / TC_HALO_W, wl = p - hl * TC_HALO_W;
        const int ph = h0 - 1 + hl, pw = w0 - 1 + wl;
        const bool inside = p < TC_HALO_W * TC_HALO_H && ph >= 0 && ph < a.H && pw >= 0 && pw < a.W && img < a.N;
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          uint32_t raw[32];
          c1.rows32(ch, stg, raw);
          if (p < TC_HALO_W * TC_HALO_H) {
            uint32_t hi[16], lo[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              float x0 = fmaxf(__uint_as_float(raw[2 * j]) + bias1_s[ch * 32 + 2 * j], 0.f);
              float x1 = fmaxf(__uint_as_float(raw[2 * j + 1]) + bias1_s[ch * 32 + 2 * j + 1], 0.f);
              if (!inside) { x0 = 0.f; x1 = 0.f; }       // conv1_2 pads its INPUT with zeros
              const __nv_bfloat16 h0b = __float2bfloat16_rn(x0), h1b = __float2bfloat16_rn(x1);
              __nv_bfloat162 hv(h0b, h1b);
              hi[j] = *reinterpret_cast<uint32_t*>(&hv);
              lo[j] = pack_bf16x2(x0 - __bfloat162float(h0b), x1 - __bfloat162float(h1b));
            }
            uint8_t* rh = halo + p * 128;
            uint8_t* rl = rh + TC_HALO_PLANE;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const int pos = ((ch * 4 + j) ^ (p & 7)) * 16;
              *reinterpret_cast<uint4*>(rh + pos) = make_uint4(hi[4 * j], hi[4 * j + 1], hi[4 * j + 2], hi[4 * j + 3]);
              *reinterpret_cast<uint4*>(rl + pos) = make_uint4(lo[4 * j], lo[4 * j + 1], lo[4 * j + 2], lo[4 * j + 3]);
            }
          }
        }
      }
      fence_proxy_async();                               // generic-proxy writes of the halo -> visible to the tensor core
      wg_sync();                                         // every halo row is written
      // C2: conv1_2 over the nine tap views of the halo tile
      Acc128<64> acc;
      int prev = -1;
      for (int tap = 0; tap < 9; ++tap) {
        mbar_wait(&w_full[stage], phase);
        const uint32_t toff = (uint32_t)((tap / 3) * TC_HALO_W + tap % 3) * 128u;
        const uint64_t a_hi = kHaloDesc | (uint64_t)(((ha + toff) >> 4) & 0x3fffu);
        const uint64_t a_lo = kHaloDesc | (uint64_t)(((ha + TC_HALO_PLANE + toff) >> 4) & 0x3fffu);
        const uint32_t sb = smem_u32(w2 + stage * F1_W2_STAGE);
        const uint64_t b_hi = gmma_desc_kmajor_sw128(sb), b_lo = gmma_desc_kmajor_sw128(sb + F1_W2_STAGE / 2);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) {
          const uint64_t ko = (uint64_t)(k * 2);
          acc.mma(a_lo + ko, a_lo + kHaloHalf + ko, b_hi + ko, (tap > 0 || k > 0) ? 1u : 0u);
          acc.mma(a_hi + ko, a_hi + kHaloHalf + ko, b_lo + ko, 1u);
          acc.mma(a_hi + ko, a_hi + kHaloHalf + ko, b_hi + ko, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&w_empty[prev]);
        prev = stage;
        if (++stage == F1_W2_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      acc.fence_operands();
      if (lane == 0) mbar_arrive(&w_empty[prev]);
      conv_epilogue_tile<64>(a, acc, stg, img, h0, w0, 0, 0, r, c, 8);
    }
  } else {
    // ================= builders: im2col rows of conv1_1 for the 180 halo pixels =================
    const int bw = warp - 5;
    int it = 0;
    for (int tile = blockIdx.x; tile < a.total_tiles; tile += gridDim.x, ++it) {
      int img, h0, w0;
      coords(tile, img, h0, w0);
      float v[2][32];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
        for (int k = 0; k < 32; ++k) v[mt][k] = 0.f;
        const int p = mt * 128 + bw * 32 + lane;
        const int hl = p / TC_HALO_W, wl = p - hl * TC_HALO_W;
        const int ph = h0 - 1 + hl, pw = w0 - 1 + wl;
        if (p < TC_HALO_W * TC_HALO_H && ph >= 0 && ph < a.H && pw >= 0 && pw < a.W && img < a.N) {
          const float* xb = fa.x + (long long)img * 3 * HW;
#pragma unroll
          for (int tap = 0; tap < 9; ++tap) {
            const int ih = ph + tap / 3 - 1, iw = pw + tap % 3 - 1;
            if (ih >= 0 && ih < a.H && iw >= 0 && iw < a.W) {
              const long long o = (long long)ih * a.W + iw;
#pragma unroll
              for (int c = 0; c < 3; ++c) v[mt][tap * 3 + c] = __ldg(xb + c * HW + o);
            }
          }
        }
      }
      mbar_wait(a1_empty, (it & 1) ^ 1);                // C1 of the previous tile has consumed A1
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int p = mt * 128 + bw * 32 + lane;
        uint8_t* rh = a1 + p * 128;
        uint8_t* rl = rh + F1_A1_PLANE;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float x0 = v[mt][8 * j + 2 * e], x1 = v[mt][8 * j + 2 * e + 1];
            const __nv_bfloat16 h0b = __float2bfloat16_rn(x0), h1b = __float2bfloat16_rn(x1);
            __nv_bfloat162 hv(h0b, h1b);
            hi[e] = *reinterpret_cast<uint32_t*>(&hv);
            lo[e] = pack_bf16x2(x0 - __bfloat162float(h0b), x1 - __bfloat162float(h1b));
          }
          const int pos = (j ^ (p & 7)) * 16;
          *reinterpret_cast<uint4*>(rh + pos) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          *reinterpret_cast<uint4*>(rl + pos) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(a1_full);
    }
  }
}

// x [N,3,H,W] fp32 -> conv1_1 -> ReLU -> conv1_2 -> ReLU -> 2x2 max-pool as hi/lo planes [N,H/2,W/2,64]
int launch_conv1_fused_tc(const float* x_nchw, const float* w1_oihw, const float* bias1, const ConvParams& p2, int N, int H,
                          int W, __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, cudaStream_t s) {
  IBL_REQUIRE(p2.w_hi && p2.w_lo && p2.bias, "fused conv1: conv1_2 weights were not re-laid-out");
  Conv1FusedArgs fa{};
  fa.x = x_nchw; fa.w1 = w1_oihw; fa.bias1 = bias1;
  ConvTcArgs& a = fa.c2;
  a.N = N; a.H = H; a.W = W; a.cin = 64; a.cout = 64;
  a.tw_log2 = 3;
  a.tiles_w = cdiv(W, 8);
  a.tiles_h = cdiv(H, 16);
  a.n_tiles = 1;
  a.total_tiles = (int)((long long)N * a.tiles_h * a.tiles_w);
  a.relu = 1; a.pool = 1;
  a.bias = p2.bias; a.y_hi = y_hi; a.y_lo = y_lo; a.y_f32 = nullptr; a.ssq = nullptr; a.ssq_stride = 0;
  a.acc_scale = tc_acc_scale(64);
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
  conv1_fused_tc_kernel<<<grid, 288, F1_SMEM, s>>>(m_whi, m_wlo, fa);
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
