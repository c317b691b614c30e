// Query x database distance + top-k, screening in ONE tensor-core pass (SURVEY 8 rows a8/a9; replaces
// pairwise_distance + np.argsort, reference ibl/evaluators.py:127-129,143, for the ranks evaluate_all reads).
//
// Round 1 screened with the bf16x3 split (3 MMAs per product) although every survivor is re-scored in exact
// fp32 anyway.  Here:
//   1. rows_f16_kernel        one pass per matrix: fp16 plane of each row scaled by a power of two (row max in
//                             [0.5,1): no overflow, 11 significant bits), exact fp32 |x|^2 (same summation order as
//                             planes_sqnorm_kernel, so the exact distances below are unchanged), the 4-norm and
//                             the max of each row (error model of the guard);
//   2. gemm_f16_top16_kernel  wgmma f16 (fp16 x fp16 -> fp32 in registers), ONE MMA per K step and 64-row
//                             half, 128 queries x 128 database rows per tile, 5-stage TMA ring, running
//                             top-16 per query in registers across the CTA's database range;
//   3. dist_finish_kernel     per query: merge of the per-range candidate lists, exact fp32 re-scoring of the 16
//                             survivors (|q|^2 + |d|^2 - 2 q.d, bit-identical to round 1's rescore_sort_kernel),
//                             final (dist, idx) sort, and the GUARD: a database row that was NOT kept has a
//                             screened distance >= s16 (the 16th screened distance); its exact distance is
//                             >= s16 - B, B = 8 sigma of the fp16 rounding error of one dot product (from the rows'
//                             4-norms) + the absolute error of fp16 subnormals.  If s16 - B < (k-th exact distance)
//                             the query is appended to a device-side list;
//   4. dist_exact_chunk_kernel / dist_exact_merge_kernel   listed queries (none, in practice: the k-th to 16th gap
//                             is ~50 B for descriptor-like data) are ranked again by exact fp32 brute force,
//                             without any host round trip: the kernels size their work from the device counter.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace ibl {

using namespace tc;

// ---- 1. fp16 planes -----------------------------------------------------------------------------
// aux[r] = {|x|^2 (exact fp32), 2^e (x = plane * 2^e), (sum x^4)^(1/4), max|x|}
__global__ void __launch_bounds__(256)
rows_f16_kernel(const float* __restrict__ x, int D, __half* __restrict__ plane, float4* __restrict__ aux) {
  __shared__ float red[8], red4[8], redm[8];
  __shared__ float scale_s;
  const long long r = blockIdx.x;
  const float4* p = reinterpret_cast<const float4*>(x + r * D);
  float ss = 0.f, s4 = 0.f, mx = 0.f;
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) {
    const float4 v = __ldg(p + i);
    ss = fmaf(v.x, v.x, ss); ss = fmaf(v.y, v.y, ss); ss = fmaf(v.z, v.z, ss); ss = fmaf(v.w, v.w, ss);
    const float a = v.x * v.x, b = v.y * v.y, c = v.z * v.z, d = v.w * v.w;
    s4 = fmaf(a, a, s4); s4 = fmaf(b, b, s4); s4 = fmaf(c, c, s4); s4 = fmaf(d, d, s4);
    mx = fmaxf(fmaxf(mx, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
    s4 += __shfl_xor_sync(0xffffffffu, s4, o);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = ss; red4[threadIdx.x >> 5] = s4; redm[threadIdx.x >> 5] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f, tot4 = 0.f, m = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { tot += red[i]; tot4 += red4[i]; m = fmaxf(m, redm[i]); }
    int e = 0;
    if (m > 0.f && m < INFINITY) frexpf(m, &e);       // m = f * 2^e, f in [0.5, 1)
    const float sc = ldexpf(1.f, e);
    scale_s = ldexpf(1.f, -e);
    aux[r] = make_float4(tot, sc, sqrtf(sqrtf(tot4)), m);
  }
  __syncthreads();
  const float inv = scale_s;
  uint2* ph = reinterpret_cast<uint2*>(plane + r * D);
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) {   // second read of the row: L1/L2 hits
    const float4 v = __ldg(p + i);
    const __half2 a = __floats2half2_rn(v.x * inv, v.y * inv), b = __floats2half2_rn(v.z * inv, v.w * inv);
    ph[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
  }
}

// max over the database rows of (4-norm, max|x|, |x|^2): the guard's bound for rows that were not kept
__global__ void dist_colmax_kernel(const float4* __restrict__ aux, int n, float* __restrict__ out3) {
  float a = 0.f, b = 0.f, c = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 v = __ldg(aux + i);
    a = fmaxf(a, v.z);
    b = fmaxf(b, v.w);
    c = fmaxf(c, v.x);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
    b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, o));
    c = fmaxf(c, __shfl_xor_sync(0xffffffffu, c, o));
  }
  if ((threadIdx.x & 31) == 0) {     // non-negative floats order like their bit patterns
    atomicMax(reinterpret_cast<int*>(out3), __float_as_int(a));
    atomicMax(reinterpret_cast<int*>(out3) + 1, __float_as_int(b));
    atomicMax(reinterpret_cast<int*>(out3) + 2, __float_as_int(c));
  }
}

// ---- 2. screening GEMM (fp16 wgmma) ----------------------------------------------------------------
struct Dist1Args {
  int M, N, K;
  int n_tiles, nt_per_item, items_per_mtile, total_items, n_valid;
  const float4* a_aux;  // per query  {|q|^2, 2^eq, ...}
  const float4* b_aux;  // per db row {|d|^2, 2^ed, ...}
  float* cand_d;        // [items_per_mtile][M][16] screened distances
  int* cand_i;          // [items_per_mtile][M][16] local database rows (-1: none)
  unsigned* gate;       // [M] orderable bits of the smallest 16th-best distance any work item of this query has reached
};

__device__ __forceinline__ uint32_t d1_ord(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float d1_unord(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__device__ __forceinline__ void d1_sts64(uint32_t addr, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ float2 d1_lds64(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}

constexpr int D1_BN = 128, D1_BK = 64;
constexpr int D1_PEND = 32;                            // pending candidates per row between two merges (see the epilogue)
constexpr int D1_A_BYTES = 128 * D1_BK * 2;            // 16 KiB: this CTA's 128 query rows
constexpr int D1_B_BYTES = D1_BN * D1_BK * 2;          // 16 KiB: one 128-row database tile
constexpr int D1_STAGES = 5;
constexpr int D1_STAGE = D1_A_BYTES + D1_B_BYTES;
constexpr int D1_BARS = 256;                           // mbarriers
constexpr int D1_BSTAGE = 4 * 32 * 8;                  // per consumer warp: {|d|^2, 2^e} of the 32 columns of a chunk
constexpr int D1_PENDB = 128 * D1_PEND * 8;            // per query row: D1_PEND pending (distance, column) pairs
constexpr int D1_SMEM = D1_STAGES * D1_STAGE + ACC_STG_BYTES + D1_BARS + D1_BSTAGE + D1_PENDB + 1024;
static_assert(D1_SMEM <= 232448, "shared-memory budget of the screening kernel");

// What bounded this kernel (profiled on the previous generation's tensor cores): the EPILOGUE.  At 10 k database rows
// per query a sorted insertion per column ran for half of all columns (any of a warp's 32 rows inserting) at ~110
// instructions a time.  The pending-list epilogue below brings it to the MMA/L2 bound.
__global__ void __launch_bounds__(160, 1)
gemm_f16_top16_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                      const Dist1Args g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* stg = reinterpret_cast<float*>(smem + D1_STAGES * D1_STAGE);
  uint8_t* tail = smem + D1_STAGES * D1_STAGE + ACC_STG_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(tail);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + D1_STAGES;       // one arrival per consumer warp
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 4 && lane == 0) {
    tma_prefetch_desc(&tm_a); tma_prefetch_desc(&tm_b);
    for (int i = 0; i < D1_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();

  auto decode = [&](int item, int& mt, int& nt0, int& ntn) {
    mt = item / g.items_per_mtile;
    const int sub = item - mt * g.items_per_mtile;
    nt0 = sub * g.nt_per_item;
    ntn = (nt0 + g.nt_per_item <= g.n_tiles) ? g.nt_per_item : (g.n_tiles - nt0);
  };
  const int kiters = g.K / D1_BK;

  if (warp == 4) {
    // TMA producer: convergent warp, one elected lane issues, warp-uniform operands
    const uint32_t smem_a = warp_uniform(smem_u32(smem));
    const uint32_t bars_a = smem_a + D1_STAGES * D1_STAGE + ACC_STG_BYTES;
    const uint32_t full_a = bars_a, empty_a = bars_a + 8 * D1_STAGES;
    int stage = 0; uint32_t phase = 0;
    for (int item = blockIdx.x; item < g.total_items; item += gridDim.x) {
      int mt, nt0, ntn;
      decode(item, mt, nt0, ntn);
      const int row0 = (int)warp_uniform((uint32_t)(mt * 128));
      for (int nt = nt0; nt < nt0 + ntn; ++nt) {
        const int col0 = (int)warp_uniform((uint32_t)(nt * D1_BN));
        for (int kit = 0; kit < kiters; ++kit) {
          const uint32_t sg = warp_uniform((uint32_t)stage);
          mbar_wait_warp_a(empty_a + 8 * sg, phase ^ 1);
          const uint32_t st = smem_a + sg * D1_STAGE, fb = full_a + 8 * sg;
          const int k0 = (int)warp_uniform((uint32_t)(kit * D1_BK));
          if (elect_one()) {
            mbar_arrive_expect_tx_a(fb, D1_STAGE);
            tma_load_2d_a(st, &tm_a, fb, k0, row0);
            tma_load_2d_a(st + D1_A_BYTES, &tm_b, fb, k0, col0);   // rows beyond the matrix are zero-filled
          }
          __syncwarp();
          if (++stage == D1_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // Consumer warpgroup: fp16 wgmma main loop, then one thread per query row.  The per-column work is scale + compare
    // + a predicated 8-byte shared-memory append to a per-row pending list; the lists are merged into the sorted top-16
    // in a compact loop (trip count = the longest list of the warp) when one could overflow within the next 16 columns,
    // and at the end of every tile.  All 32 rows of a warp insert side by side in that loop, so the walk runs once per
    // ~16 appended candidates of the fullest row instead of once per column with a candidate anywhere.
    const int q = warp;
    const int rloc = threadIdx.x;
    const uint32_t smem_a = smem_u32(smem);
    // shared-state-space addresses (the generic pointer arithmetic above makes the compiler emit generic LD/ST)
    const uint32_t bst = smem_u32(tail + D1_BARS) + q * 256;
    const uint32_t pend = smem_u32(tail + D1_BARS + D1_BSTAGE) + rloc * 8;   // [slot][128 rows] x 8 B
    int stage = 0; uint32_t phase = 0;
    for (int item = blockIdx.x; item < g.total_items; item += gridDim.x) {
      int mt, nt0, ntn;
      decode(item, mt, nt0, ntn);
      const int row = mt * 128 + rloc;
      const bool row_ok = row < g.M;
      float an = 0.f, m2sa = 0.f;
      if (row_ok) { const float4 t = __ldg(g.a_aux + row); an = t.x; m2sa = -2.f * t.y; }
      float td[16];
      int ti[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) { td[j] = INFINITY; ti[j] = -1; }
      uint32_t paddr = pend;                               // next free slot of this row's pending list
      float thr = row_ok ? INFINITY : -INFINITY;           // rows beyond the matrix never append
      // merge this row's pending list into the sorted top-16; the 32 rows of the warp run the loop together
      auto merge_pending = [&]() {
        const int cnt = (int)((paddr - pend) >> 10);
        const int longest = __reduce_max_sync(0xffffffffu, cnt);
#pragma unroll 1
        for (int e = 0; e < longest; ++e) {
          if (e < cnt) {
            const float2 v = d1_lds64(pend + e * 1024);
            const float d = v.x;
            if (d < td[15]) {
              const int col = __float_as_int(v.y);
              // Sorted insert without a dependency chain: the slot is counted with 16 independent compares and every
              // entry is rewritten from the OLD values of itself and its left neighbour (descending s).
              int pos = 0;
#pragma unroll
              for (int s = 0; s < 16; ++s) pos += (td[s] <= d) ? 1 : 0;
#pragma unroll
              for (int s = 15; s > 0; --s) {
                const bool shift = s > pos, here = s == pos;
                td[s] = shift ? td[s - 1] : (here ? d : td[s]);
                ti[s] = shift ? ti[s - 1] : (here ? col : ti[s]);
              }
              if (pos == 0) { td[0] = d; ti[0] = col; }
            }
          }
        }
        paddr = pend;
      };
      for (int nt = nt0; nt < nt0 + ntn; ++nt) {
        // Shared gate: the work items of one query block scan different database ranges concurrently, each keeping its
        // own top-16.  An element that is not below the 16th-best distance ANY of them has already reached cannot be in
        // the merged top-16, so every item publishes its 16th-best (atomicMin) after each tile and reads the common
        // value before the next: the gate tightens with the UNION of the columns scanned so far.  A stale read only
        // costs efficiency.  Ties at the gate are dropped: the guard's error bound covers them.
        if (row_ok) {
          const unsigned gv = *reinterpret_cast<volatile unsigned*>(g.gate + row);
          if (gv != 0xFFFFFFFFu) thr = fminf(thr, d1_unord(gv));       // 0xFFFFFFFF = "no gate yet" (the memset pattern)
        }
        Acc128<D1_BN> acc;
        int prev = -1;
        for (int kit = 0; kit < kiters; ++kit) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_a + stage * D1_STAGE;
          const uint64_t da = gmma_desc_kmajor_sw128(sa), db = gmma_desc_kmajor_sw128(sa + D1_A_BYTES);
          constexpr uint64_t kHalf = 64 * 128 / 16;   // query rows 64-127: +8 KiB
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < D1_BK / 16; ++k)
            acc.mma<true>(da + (uint64_t)(k * 2), da + kHalf + (uint64_t)(k * 2), db + (uint64_t)(k * 2),
                          (kit > 0 || k > 0) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
          prev = stage;
          if (++stage == D1_STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        acc.fence_operands();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
#pragma unroll
        for (int ch = 0; ch < D1_BN / 32; ++ch) {     // unrolled: the accumulator is indexed with constants only
          const int col0 = nt * D1_BN + ch * 32;
          if (col0 >= g.n_valid) break;                    // block-uniform: the rest of the tile is padding
          // The per-column terms {|d|^2, 2^e} of this chunk: ONE coalesced load (lane j fetches column col0 + j) staged
          // in shared memory and read back as warp-wide broadcasts, instead of a chain of dependent per-column loads.
          float2 mine = make_float2(INFINITY, 0.f);        // padding columns: +inf, never below the threshold
          if (col0 + lane < g.n_valid) { const float4 t = __ldg(g.b_aux + col0 + lane); mine = make_float2(t.x, t.y); }
          uint32_t raw[32];
          acc.rows32(ch, stg, raw);
          __syncwarp();                                    // the previous chunk's broadcast reads are done
          d1_sts64(bst + lane * 8, mine.x, mine.y);
          __syncwarp();
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (__any_sync(0xffffffffu, paddr > pend + (D1_PEND - 16) * 1024)) {   // could overflow within 16 columns: merge first
              merge_pending();
              thr = fminf(thr, td[15]);
            }
            float2 c[16];
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) c[jj] = d1_lds64(bst + (h * 16 + jj) * 8);   // issued back to back
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) {
              const int j = h * 16 + jj;
              const float d = fmaf(m2sa * c[jj].y, __uint_as_float(raw[j]), an + c[jj].x);
              if (d < thr) { d1_sts64(paddr, d, __int_as_float(col0 + j)); paddr += 1024; }
            }
          }
        }
        merge_pending();
        if (row_ok && td[15] < thr) {
          thr = td[15];
          atomicMin(g.gate + row, d1_ord(thr));
        }
      }
      if (row_ok) {
        const int sub = item % g.items_per_mtile;
        float4* od = reinterpret_cast<float4*>(g.cand_d + ((long long)sub * g.M + row) * 16);
        int4* oi = reinterpret_cast<int4*>(g.cand_i + ((long long)sub * g.M + row) * 16);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          od[j] = make_float4(td[4 * j], td[4 * j + 1], td[4 * j + 2], td[4 * j + 3]);
          oi[j] = make_int4(ti[4 * j], ti[4 * j + 1], ti[4 * j + 2], ti[4 * j + 3]);
        }
      }
    }
  }
}

// ---- 3. merge + exact re-scoring + sort + guard ---------------------------------------------------------

// exact distance of query row (staged at qrow) and database row ci, one warp; same arithmetic as round 1's
// rescore_sort_kernel: lane-strided float4 FMAs, xor-shuffle tree, fmaf(-2, dot, |q|^2 + |d|^2)
__device__ __forceinline__ float d1_exact(const float* qrow, const float* __restrict__ dp, int d, int lane, float an,
                                          float bn) {
  float acc = 0.f;
  for (int i = lane * 4; i < d; i += 128) {
    const float4 a = *reinterpret_cast<const float4*>(qrow + i);
    const float4 b = __ldg(reinterpret_cast<const float4*>(dp + i));
    acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
    acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return fmaf(-2.f, acc, an + bn);
}

struct FinishArgs {
  const float* q; const float* db;
  const float4* q_aux; const float4* db_aux;
  const float* db_max2;          // {max 4-norm, max |x|, max |x|^2} over the database rows
  const float* cand_d; const int* cand_i;
  int m, d, runs, k_out, n_valid;
  long long idx_base;
  float* out_dist; long long* out_idx;
  int* flag_count; int* flag_list;
};

// kappa = 8 standard deviations; rms relative rounding error of fp16 RN = 2^-11 * 0.41; two operands (sqrt 2);
// distance = -2 dot (factor 2)  ->  8 * 2 * 1.414 * 0.41 * 2^-11
#define D1_GUARD_C (8.f * 2.f * 1.41421356f * 0.41f * 4.8828125e-4f)

__global__ void __launch_bounds__(128)
dist_finish_kernel(const FinishArgs g) {
  extern __shared__ __align__(16) float qs[];   // [d] when it fits
  __shared__ unsigned long long keys[128];
  __shared__ unsigned long long skeys[128];
  const long long row = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int d = g.d;
  const bool staged = d <= 16384;
  if (staged) {
    for (int i = threadIdx.x * 4; i < d; i += 128 * 4)
      *reinterpret_cast<float4*>(qs + i) = __ldg(reinterpret_cast<const float4*>(g.q + row * d + i));
  }
  const float* qrow = staged ? qs : (g.q + row * d);
  // ---- merge: the 16 best screened candidates of runs x 16 (runs <= 8) ----
  const int total = g.runs * 16;
  {
    unsigned long long key = ~0ull;
    if ((int)threadIdx.x < total) {
      const int r = threadIdx.x >> 4, j = threadIdx.x & 15;
      const long long src = ((long long)r * g.m + row) * 16 + j;
      const int ci = g.cand_i[src];
      if (ci >= 0) key = ((unsigned long long)d1_ord(g.cand_d[src]) << 32) | (unsigned)ci;
    }
    skeys[threadIdx.x] = key;
  }
  for (int size = 2; size <= 128; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      if (threadIdx.x < 64) {
        const int i = threadIdx.x;
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long a = skeys[lo], b = skeys[hi];
        if ((a > b) == up) { skeys[lo] = b; skeys[hi] = a; }
      }
    }
  }
  __syncthreads();
  const float4 qa = __ldg(g.q_aux + row);
  // ---- exact fp32 re-scoring of the 16 survivors ----
  for (int c = wid; c < 128; c += 4) {
    unsigned long long key = ~0ull;
    if (c < 16) {
      const unsigned long long sk = skeys[c];
      if (sk != ~0ull) {
        const long long ci = (long long)(uint32_t)(sk & 0xffffffffu);
        const float dist = d1_exact(qrow, g.db + ci * d, d, lane, qa.x, __ldg(&g.db_aux[ci].x));
        key = ((unsigned long long)d1_ord(dist) << 32) | (unsigned)ci;
      }
    }
    if (lane == 0) keys[c] = key;
  }
  for (int size = 2; size <= 16; size <<= 1) {          // only keys[0..15] can be valid
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      if (threadIdx.x < 8) {
        const int i = threadIdx.x;
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long a = keys[lo], b = keys[hi];
        if ((a > b) == up) { keys[lo] = b; keys[hi] = a; }
      }
    }
  }
  __syncthreads();
  if ((int)threadIdx.x < g.k_out) {
    const unsigned long long key = keys[threadIdx.x];
    if (key == ~0ull) {
      g.out_dist[row * g.k_out + threadIdx.x] = INFINITY;
      g.out_idx[row * g.k_out + threadIdx.x] = -1;
    } else {
      g.out_dist[row * g.k_out + threadIdx.x] = d1_unord((uint32_t)(key >> 32));
      g.out_idx[row * g.k_out + threadIdx.x] = g.idx_base + (long long)(uint32_t)(key & 0xffffffffu);
    }
  }
  // ---- guard ----
  if (threadIdx.x == 0 && g.n_valid > 16) {              // with <= 16 rows everything was re-scored
    const unsigned long long s16k = skeys[15];
    const int kk = g.k_out < 16 ? g.k_out : 16;
    const unsigned long long ek = keys[kk - 1];
    bool flag = (s16k == ~0ull) || (ek == ~0ull);        // cannot happen with n_valid > 16; be safe
    if (!flag) {
      const float s16 = d1_unord((uint32_t)(s16k >> 32)), e_k = d1_unord((uint32_t)(ek >> 32));
      // statistical part: 8 sigma of the fp16 rounding error of one dot product (Cauchy-Schwarz on the 4-norms);
      // absolute part: values below 2^-14 of the row max are fp16 subnormals, error <= 2^-24 * row max each:
      // |dot error| <= 2^-24 sqrt(D) (dmax |q| + qmax |d|), distance = -2 dot
      const float bound = D1_GUARD_C * qa.z * __ldg(g.db_max2) +
                          2.f * 5.9604645e-8f * sqrtf((float)d) *
                              (__ldg(g.db_max2 + 1) * sqrtf(qa.x) + qa.w * sqrtf(__ldg(g.db_max2 + 2)));
      flag = !(s16 - bound > e_k);                       // also catches NaN
    }
    if (flag) g.flag_list[atomicAdd(g.flag_count, 1)] = (int)row;
  }
}

// ---- 4. exact brute force for the listed queries ----------------------------------------------------
constexpr int DX_CHUNK = 4096;    // database rows per work item

struct ExactArgs {
  const float* q; const float* db;
  const float4* q_aux; const float4* db_aux;
  int m, d, n_valid, k, nchunks;
  long long idx_base;
  const int* flag_count; const int* flag_list;
  unsigned long long* scratch;   // [m][nchunks][16] keys
  float* out_dist; long long* out_idx;
};

// work item = (listed query f, chunk c): exact distances of DX_CHUNK rows, the 16 smallest keys to scratch
__global__ void __launch_bounds__(256)
dist_exact_chunk_kernel(const ExactArgs g) {
  extern __shared__ __align__(16) float qs[];
  __shared__ unsigned long long best[8][16];
  const int count = *g.flag_count;
  const int items = count * g.nchunks;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const bool staged = g.d <= 16384;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int f = item / g.nchunks, c = item - f * g.nchunks;
    const long long row = g.flag_list[f];
    __syncthreads();
    if (staged)
      for (int i = threadIdx.x * 4; i < g.d; i += 256 * 4)
        *reinterpret_cast<float4*>(qs + i) = __ldg(reinterpret_cast<const float4*>(g.q + row * g.d + i));
    __syncthreads();
    const float* qrow = staged ? qs : (g.q + row * g.d);
    const float an = __ldg(&g.q_aux[row].x);
    unsigned long long mine[16];               // this warp's 16 best (every lane holds the same list)
#pragma unroll
    for (int j = 0; j < 16; ++j) mine[j] = ~0ull;
    const int j0 = c * DX_CHUNK, j1 = min(g.n_valid, j0 + DX_CHUNK);
    for (int j = j0 + wid; j < j1; j += 8) {
      const float dist = d1_exact(qrow, g.db + (long long)j * g.d, g.d, lane, an, __ldg(&g.db_aux[j].x));
      unsigned long long key = ((unsigned long long)d1_ord(dist) << 32) | (unsigned)j;
      if (key < mine[15]) {
        mine[15] = key;
#pragma unroll
        for (int s = 15; s > 0; --s)
          if (mine[s] < mine[s - 1]) { const unsigned long long t = mine[s]; mine[s] = mine[s - 1]; mine[s - 1] = t; }
      }
    }
    if (lane == 0)
#pragma unroll
      for (int j = 0; j < 16; ++j) best[wid][j] = mine[j];
    __syncthreads();
    if (threadIdx.x == 0) {                    // 16 smallest of the 8 sorted lists (rare path: serial merge)
      int head[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      unsigned long long* out = g.scratch + ((long long)row * g.nchunks + c) * 16;
      for (int t = 0; t < 16; ++t) {
        int bw = 0;
        unsigned long long bk = ~0ull;
        for (int w = 0; w < 8; ++w)
          if (head[w] < 16 && best[w][head[w]] < bk) { bk = best[w][head[w]]; bw = w; }
        out[t] = bk;
        if (bk != ~0ull) ++head[bw];
      }
    }
  }
}

// one block per listed query: merge its nchunks x 16 keys, write the final top-k over the guarded result
__global__ void __launch_bounds__(128)
dist_exact_merge_kernel(const ExactArgs g) {
  const int count = *g.flag_count;
  for (int f = blockIdx.x; f < count; f += gridDim.x) {
    const long long row = g.flag_list[f];
    const unsigned long long* src = g.scratch + row * g.nchunks * 16;
    if (threadIdx.x == 0) {                    // rare path: a serial k-way selection is fine
      unsigned long long prev = 0;
      bool first = true;
      for (int t = 0; t < g.k; ++t) {
        unsigned long long bk = ~0ull;
        for (int i = 0; i < g.nchunks * 16; ++i) {
          const unsigned long long key = src[i];
          if ((first || key > prev) && key < bk) bk = key;
        }
        if (bk == ~0ull) {
          g.out_dist[row * g.k + t] = INFINITY;
          g.out_idx[row * g.k + t] = -1;
        } else {
          g.out_dist[row * g.k + t] = d1_unord((uint32_t)(bk >> 32));
          g.out_idx[row * g.k + t] = g.idx_base + (long long)(uint32_t)(bk & 0xffffffffu);
        }
        prev = bk;
        first = false;
      }
    }
  }
}

// ---- host -----------------------------------------------------------------------------------------
static int pick_runs1(int m_tiles, int n_tiles) {
  const int G = device_sm_count();
  int best = 1;
  double best_eff = -1.0;
  for (int r = 1; r <= n_tiles && r <= 8; ++r) {          // dist_finish_kernel merges up to 8 x 16 candidates
    const int per = cdiv(n_tiles, r), runs = cdiv(n_tiles, per);
    const long long total = (long long)m_tiles * runs, waves = (total + G - 1) / G;
    const double eff = (double)m_tiles * n_tiles / ((double)waves * G * per);
    if (eff > best_eff + 1e-9) { best_eff = eff; best = runs; }
  }
  return best;
}

size_t dist1_workspace_bytes(int m, int n, int d, size_t* off /*[8]*/) {
  // layout: q plane | db plane | q aux | db aux | db max2 + flag count (256 B) | flag list | cand_d | cand_i | scratch
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += (bytes + 255) & ~(size_t)255; return at; };
  off[0] = take((size_t)m * d * 2);
  off[1] = take((size_t)n * d * 2);
  off[2] = take((size_t)m * 16);
  off[3] = take((size_t)n * 16);
  off[4] = take(256);
  off[5] = take((size_t)m * 4 + (size_t)m * 4);     // guard list | shared gates
  off[6] = take((size_t)8 * m * 16 * 4);
  off[7] = take((size_t)8 * m * 16 * 4);
  const int nchunks = cdiv(n > 0 ? n : 1, DX_CHUNK);
  off[8] = take((size_t)m * nchunks * 16 * 8);
  return o;
}

// q [m,d], db [n,d] fp32 (device); n_valid <= n; k <= 12.  ws: dist1_workspace_bytes(m, n, d).
int launch_dist_topk_1pass(const float* q, int m, const float* db, int n, int n_valid, int d, int k, long long idx_base,
                           void* ws, float* out_dist, long long* out_idx, uint64_t* launches, cudaStream_t s) {
  IBL_REQUIRE(d % 64 == 0 && k >= 1 && k <= 12 && n_valid >= 1, "1-pass distance: d % 64 == 0, 1 <= k <= 12");
  size_t off[9];
  dist1_workspace_bytes(m, n, d, off);
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  __half* qp = reinterpret_cast<__half*>(w + off[0]);
  __half* dp = reinterpret_cast<__half*>(w + off[1]);
  float4* qa = reinterpret_cast<float4*>(w + off[2]);
  float4* da = reinterpret_cast<float4*>(w + off[3]);
  float* dmax2 = reinterpret_cast<float*>(w + off[4]);
  int* fcount = reinterpret_cast<int*>(w + off[4] + 16);
  int* flist = reinterpret_cast<int*>(w + off[5]);
  unsigned* gate = reinterpret_cast<unsigned*>(w + off[5] + (size_t)m * 4);
  float* cd = reinterpret_cast<float*>(w + off[6]);
  int* ci = reinterpret_cast<int*>(w + off[7]);
  unsigned long long* scratch = reinterpret_cast<unsigned long long*>(w + off[8]);

  IBL_CUDA_OK(cudaMemsetAsync(w + off[4], 0, 32, s));
  IBL_CUDA_OK(cudaMemsetAsync(gate, 0xFF, (size_t)m * 4, s));      // orderable +max: no gate yet
  rows_f16_kernel<<<m, 256, 0, s>>>(q, d, qp, qa);
  rows_f16_kernel<<<n, 256, 0, s>>>(db, d, dp, da);
  dist_colmax_kernel<<<cdiv(n_valid, 256) < 64 ? cdiv(n_valid, 256) : 64, 256, 0, s>>>(da, n_valid, dmax2);
  IBL_CUDA_OK(cudaGetLastError());

  CUtensorMap ma, mb;
  {
    uint64_t dims_a[2] = {(uint64_t)d, (uint64_t)m}, dims_b[2] = {(uint64_t)d, (uint64_t)n};
    uint64_t str[1] = {(uint64_t)d * 2};
    uint32_t box[2] = {64, 128};
    IBL_RET(make_tmap(&ma, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, qp, dims_a, str, box));
    IBL_RET(make_tmap(&mb, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, dp, dims_b, str, box));
  }
  Dist1Args g{};
  g.M = m; g.N = n; g.K = d;
  g.n_tiles = cdiv(n_valid, D1_BN);
  const int m_tiles = cdiv(m, 128);
  const int runs = pick_runs1(m_tiles, g.n_tiles);
  g.nt_per_item = cdiv(g.n_tiles, runs);
  g.items_per_mtile = cdiv(g.n_tiles, g.nt_per_item);
  g.total_items = m_tiles * g.items_per_mtile;
  g.n_valid = n_valid;
  g.a_aux = qa; g.b_aux = da; g.cand_d = cd; g.cand_i = ci; g.gate = gate;
  static DeviceOnce attr_done;   // the attributes are per device
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(gemm_f16_top16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, D1_SMEM));
    IBL_CUDA_OK(cudaFuncSetAttribute(dist_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    IBL_CUDA_OK(cudaFuncSetAttribute(dist_exact_chunk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    attr_done.mark();
  }
  const int sms = device_sm_count();
  gemm_f16_top16_kernel<<<g.total_items < sms ? g.total_items : sms, 160, D1_SMEM, s>>>(ma, mb, g);
  IBL_CUDA_OK(cudaGetLastError());

  FinishArgs f{};
  f.q = q; f.db = db; f.q_aux = qa; f.db_aux = da; f.db_max2 = dmax2; f.cand_d = cd; f.cand_i = ci;
  f.m = m; f.d = d; f.runs = g.items_per_mtile; f.k_out = k; f.n_valid = n_valid; f.idx_base = idx_base;
  f.out_dist = out_dist; f.out_idx = out_idx; f.flag_count = fcount; f.flag_list = flist;
  const size_t qsm = d <= 16384 ? (size_t)d * sizeof(float) : 16;
  dist_finish_kernel<<<m, 128, qsm, s>>>(f);
  IBL_CUDA_OK(cudaGetLastError());

  ExactArgs x{};
  x.q = q; x.db = db; x.q_aux = qa; x.db_aux = da; x.m = m; x.d = d; x.n_valid = n_valid; x.k = k;
  x.nchunks = cdiv(n_valid, DX_CHUNK); x.idx_base = idx_base; x.flag_count = fcount; x.flag_list = flist;
  x.scratch = scratch; x.out_dist = out_dist; x.out_idx = out_idx;
  dist_exact_chunk_kernel<<<device_sm_count() * 2, 256, qsm, s>>>(x);     // exits at once when nothing is listed
  dist_exact_merge_kernel<<<32, 128, 0, s>>>(x);
  IBL_CUDA_OK(cudaGetLastError());
  if (launches) *launches += 7;
  return IBL_OK;
}

// test hook: number of queries the guard listed in the last call on this workspace (synchronises)
int dist1_last_flag_count(void* ws, int m, int n, int d, int* out, cudaStream_t s) {
  size_t off[9];
  dist1_workspace_bytes(m, n, d, off);
  IBL_CUDA_OK(cudaMemcpyAsync(out, reinterpret_cast<uint8_t*>(ws) + off[4] + 16, sizeof(int), cudaMemcpyDeviceToHost, s));
  IBL_CUDA_OK(cudaStreamSynchronize(s));
  return IBL_OK;
}

}  // namespace ibl
