// Query x database distance + top-k, screening in ONE tensor-core pass (SURVEY 8 rows a8/a9; replaces
// pairwise_distance + np.argsort, reference ibl/evaluators.py:127-129,143, for the ranks evaluate_all reads).
//
// Round 1 screened with the bf16x3 split (3 MMAs per product) although every survivor is re-scored in exact
// fp32 anyway.  Here:
//   1. rows_f16_kernel        one pass per matrix: fp16 plane of each row scaled by a power of two (row max in
//                             [0.5,1): no overflow, 11 significant bits), exact fp32 |x|^2 (same summation order as
//                             planes_sqnorm_kernel, so the exact distances below are unchanged) and the norm of
//                             each row's rounding residual x - 2^e plane (error model of the guard);
//   2. gemm_f16_top16_kernel  wgmma f16 (fp16 x fp16 -> fp32 in registers), ONE MMA per K step and 64-row
//                             half, 128 queries x 128 database rows per tile, 5-stage TMA ring, running
//                             top-16 per query in registers across the CTA's database range;
//   3. dist_finish_kernel     per query: merge of the per-range candidate lists, exact fp32 re-scoring of the 16
//                             survivors (|q|^2 + |d|^2 - 2 q.d, bit-identical to round 1's rescore_sort_kernel),
//                             final (dist, idx) sort, and the GUARD: a database row that was NOT kept has a
//                             screened distance >= s16 (the 16th screened distance); its exact distance is
//                             >= s16 - B, B = d1_screen_bound: a rigorous bound of the operand rounding (the rows'
//                             residual norms, Cauchy-Schwarz) + a statistical allowance for the tensor core's fp32
//                             accumulation.  If s16 - B <= (k-th exact distance) the query is appended to a
//                             device-side list;
//   4. dist_exact_scan_kernel / dist_exact_finish_kernel   listed queries (about 0.1% of retrieval-like queries at
//                             4096 dimensions, 10% at 32768, measured on synth.make_gallery) are ranked again by
//                             exact fp32 brute force, without any host round trip: the kernels size their work from
//                             the device counter, and one pass over the database serves every listed query.
//   5. dist_guard_kernel      the same guard and fallback after the bf16x3 screening of tc_gemm.cu.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"
#include "dist_exact.cuh"

namespace ibl {

using namespace tc;

// ---- 1. fp16 planes -----------------------------------------------------------------------------
// aux[r] = {|x|^2 (exact fp32), 2^e (x = plane * 2^e), |x - 2^e plane| (the rounding residual), max|x|}
__global__ void __launch_bounds__(256)
rows_f16_kernel(const float* __restrict__ x, int D, __half* __restrict__ plane, float4* __restrict__ aux) {
  __shared__ float red[8], redm[8];
  __shared__ float scale_s, sc_s, tot_s, m_s;
  const long long r = blockIdx.x;
  const float4* p = reinterpret_cast<const float4*>(x + r * D);
  float ss = 0.f, mx = 0.f;
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) {
    const float4 v = __ldg(p + i);
    ss = fmaf(v.x, v.x, ss); ss = fmaf(v.y, v.y, ss); ss = fmaf(v.z, v.z, ss); ss = fmaf(v.w, v.w, ss);
    mx = fmaxf(fmaxf(mx, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = ss; redm[threadIdx.x >> 5] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f, m = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { tot += red[i]; m = fmaxf(m, redm[i]); }
    int e = 0;
    if (m > 0.f && m < INFINITY) frexpf(m, &e);       // m = f * 2^e, f in [0.5, 1)
    scale_s = ldexpf(1.f, -e);
    sc_s = ldexpf(1.f, e);
    tot_s = tot;
    m_s = m;
  }
  __syncthreads();
  const float inv = scale_s, sc = sc_s;
  uint2* ph = reinterpret_cast<uint2*>(plane + r * D);
  float rr = 0.f;                                      // |x - 2^e plane|^2: every element's rounding, subnormals included
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) {   // second read of the row: L1/L2 hits
    const float4 v = __ldg(p + i);
    const __half2 a = __floats2half2_rn(v.x * inv, v.y * inv), b = __floats2half2_rn(v.z * inv, v.w * inv);
    ph[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
    const float2 fa = __half22float2(a), fb = __half22float2(b);
    const float r0 = v.x - fa.x * sc, r1 = v.y - fa.y * sc, r2 = v.z - fb.x * sc, r3 = v.w - fb.y * sc;
    rr = fmaf(r0, r0, rr); rr = fmaf(r1, r1, rr); rr = fmaf(r2, r2, rr); rr = fmaf(r3, r3, rr);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) rr += __shfl_xor_sync(0xffffffffu, rr, o);
  __syncthreads();                                     // red[] is reused
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = rr;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tr = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tr += red[i];
    aux[r] = make_float4(tot_s, sc, sqrtf(tr), m_s);
  }
}

// max over the database rows of (residual norm, max|x|, |x|^2): the guard's bound for rows that were not kept
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

struct FinishArgs {
  const float* q; const float* db;
  const float4* q_aux; const float4* db_aux;
  const float* db_max2;          // {max 4-norm, max |x|, max |x|^2} over the database rows
  const float* cand_d; const int* cand_i;
  int m, d, runs, k_out, n_valid;
  long long idx_base;
  float* out_dist; long long* out_idx;
  int* flag_count; int* flag_list; int* list_cnt;
};

// The guard's B: d1_screen_bound (dist_exact.cuh).

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
      // fp16 operands: no lo plane, one MMA per K step; the residuals include the subnormals' rounding
      const float bound = d1_screen_bound(qa.x, 0.f, qa.z, __ldg(g.db_max2 + 2), 0.f, __ldg(g.db_max2), d, 1);
      flag = !(s16 - bound > e_k);                       // also catches NaN
    }
    if (flag) {
      const int f = atomicAdd(g.flag_count, 1);
      g.flag_list[f] = (int)row;
      g.list_cnt[f] = 0;
    }
  }
}

// ---- 4. exact brute force for the listed queries ----------------------------------------------------
// A listed query already has k re-scored rows at exact distances <= e_k, so its true top-k lies at exact distance
// <= e_k.  One pass over the database scores every row against every listed query (the row stays in L1 across the
// queries: the database is read once however many queries are listed) and appends the rows at <= e_k to the query's
// list; a second kernel sorts each list.  A list that overflows (more than DX_CAP rows within e_k: heavy ties) is
// ranked by a blockwise scan of the whole database instead.
constexpr int DX_CAP = 256;       // listed rows per query
// byte offset of the lists after the [m] list counters (the 8-byte keys need 8-byte alignment whatever m is)
static size_t dx_lists_at(int m) { return ((size_t)m * 4 + 255) & ~(size_t)255; }

struct ExactArgs {
  const float* q; const float* db;
  const float* q_sq; const float* db_sq;   // exact fp32 |x|^2 of every row, sq_stride floats apart
  int sq_stride;
  int m, d, n_valid, k;
  long long idx_base;
  const int* flag_count; const int* flag_list;
  int* list_cnt;                 // [m] per listed query (zeroed by the guard that lists it)
  unsigned long long* lists;     // [m][DX_CAP] (dist, row) keys
  float* out_dist; long long* out_idx;
};

// Listed queries in groups of up to DX_QG staged in shared memory; one warp per database row (grid-stride), the
// row's float4 slices loaded once and multiplied into every staged query, in d1_exact's order (lane-strided FMAs,
// xor-shuffle tree, the same final fma): the distances are bit-identical to the re-scored ones.
constexpr int DX_QG = 8;
constexpr int DX_QSMEM = 128 * 1024;      // staged query rows: min(DX_QG, 32768 / d) of them
constexpr int DX_SCAN_WARPS = 16;
__global__ void __launch_bounds__(DX_SCAN_WARPS * 32)
dist_exact_scan_kernel(const ExactArgs g) {
  extern __shared__ __align__(16) float qs[];
  const int count = *g.flag_count;
  if (count == 0) return;
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * DX_SCAN_WARPS;
  const int qg = min(DX_QG, max(1, (DX_QSMEM / 4) / g.d));
  for (int f0 = 0; f0 < count; f0 += qg) {
    const int nq = min(qg, count - f0);
    __syncthreads();
    for (int t = 0; t < nq; ++t) {
      const float* src = g.q + (long long)g.flag_list[f0 + t] * g.d;
      for (int i = threadIdx.x * 4; i < g.d; i += DX_SCAN_WARPS * 32 * 4)
        *reinterpret_cast<float4*>(qs + t * g.d + i) = __ldg(reinterpret_cast<const float4*>(src + i));
    }
    __syncthreads();
    for (int j = blockIdx.x * DX_SCAN_WARPS + (threadIdx.x >> 5); j < g.n_valid; j += warps) {
      const float* dp = g.db + (long long)j * g.d;
      float acc[DX_QG];
#pragma unroll
      for (int t = 0; t < DX_QG; ++t) acc[t] = 0.f;
#pragma unroll 2
      for (int i = lane * 4; i < g.d; i += 128) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(dp + i));
#pragma unroll
        for (int t = 0; t < DX_QG; ++t) {
          if (t < nq) {
            const float4 a = *reinterpret_cast<const float4*>(qs + t * g.d + i);
            acc[t] = fmaf(a.x, b.x, acc[t]); acc[t] = fmaf(a.y, b.y, acc[t]);
            acc[t] = fmaf(a.z, b.z, acc[t]); acc[t] = fmaf(a.w, b.w, acc[t]);
          }
        }
      }
      const float bn = __ldg(g.db_sq + (long long)j * g.sq_stride);
#pragma unroll
      for (int t = 0; t < DX_QG; ++t) {
        if (t < nq) {
          float v = acc[t];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          const int f = f0 + t;
          const long long row = g.flag_list[f];
          const float dist = fmaf(-2.f, v, __ldg(g.q_sq + row * g.sq_stride) + bn);
          if (lane == 0 && dist <= g.out_dist[row * g.k + g.k - 1]) {   // e_k of the re-scored list
            const int at = atomicAdd(g.list_cnt + f, 1);
            if (at < DX_CAP) g.lists[(long long)f * DX_CAP + at] = ((unsigned long long)d1_ord(dist) << 32) | (unsigned)j;
          }
        }
      }
    }
  }
}

// the attribute is per device
static int dx_scan_attr() {
  static DeviceOnce done;
  if (!done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(dist_exact_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DX_QSMEM));
    done.mark();
  }
  return IBL_OK;
}

static size_t dx_scan_smem(int d) { return (size_t)min(DX_QG, max(1, (DX_QSMEM / 4) / d)) * d * sizeof(float); }

// 512 keys in shared memory, ascending (256 threads)
__device__ __forceinline__ void dx_sort512(unsigned long long* keys) {
  for (int size = 2; size <= 512; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      const int i = threadIdx.x;
      const int lo = 2 * i - (i & (stride - 1));
      const int hi = lo + stride;
      const bool up = ((lo & size) == 0);
      const unsigned long long a = keys[lo], b = keys[hi];
      if ((a > b) == up) { keys[lo] = b; keys[hi] = a; }
    }
  }
  __syncthreads();
}

// one block per listed query: sort its list (or, on overflow, scan the database 256 rows at a time keeping the 256
// best) and write the final top-k
__global__ void __launch_bounds__(256)
dist_exact_finish_kernel(const ExactArgs g) {
  __shared__ unsigned long long keys[512];
  const int count = *g.flag_count;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int f = blockIdx.x; f < count; f += gridDim.x) {
    const long long row = g.flag_list[f];
    const int cnt = g.list_cnt[f];
    __syncthreads();
    for (int i = threadIdx.x; i < 512; i += 256)
      keys[i] = (cnt <= DX_CAP && i < cnt) ? g.lists[(long long)f * DX_CAP + i] : ~0ull;
    __syncthreads();
    if (cnt <= DX_CAP) {
      dx_sort512(keys);
    } else {
      const float* qrow = g.q + row * g.d;
      const float an = __ldg(g.q_sq + row * g.sq_stride);
      for (int j0 = 0; j0 < g.n_valid; j0 += 256) {     // keys[0, 256): best so far; keys[256, 512): this chunk
        for (int t = wid; t < 256; t += 8) {
          const int j = j0 + t;
          unsigned long long key = ~0ull;
          if (j < g.n_valid) {
            const float dist = d1_exact(qrow, g.db + (long long)j * g.d, g.d, lane, an,
                                        __ldg(g.db_sq + (long long)j * g.sq_stride));
            key = ((unsigned long long)d1_ord(dist) << 32) | (unsigned)j;
          }
          if (lane == 0) keys[256 + t] = key;
        }
        dx_sort512(keys);
      }
    }
    if ((int)threadIdx.x < g.k) {
      const unsigned long long key = keys[threadIdx.x];
      g.out_dist[row * g.k + threadIdx.x] = key == ~0ull ? INFINITY : d1_unord((uint32_t)(key >> 32));
      g.out_idx[row * g.k + threadIdx.x] = key == ~0ull ? -1 : g.idx_base + (long long)(uint32_t)(key & 0xffffffffu);
    }
  }
}

// ---- 5. guard + exact fallback for the bf16x3 screening paths (tc_gemm.cu) -----------------------------
// max over the database rows of (|lo|, |x - hi - lo|, |x|^2)
__global__ void dist_guard_colmax_kernel(const float2* __restrict__ err, const float* __restrict__ sq, int n,
                                         float* __restrict__ out3) {
  float a = 0.f, b = 0.f, c = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float2 v = __ldg(err + i);
    a = fmaxf(a, v.x);
    b = fmaxf(b, v.y);
    c = fmaxf(c, __ldg(sq + i));
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

// one thread per query.  screened [m][kc]: the kc smallest screened distances, ascending; a row that is not among
// them has a screened distance >= the last.  Same test as dist_finish_kernel's guard, with three MMAs per K step.
__global__ void dist_guard_kernel(const float* __restrict__ screened, int kc, const float* __restrict__ q_sq,
                                  const float2* __restrict__ q_err, const float* __restrict__ db_max3,
                                  const float* __restrict__ out_dist, int k, int m, int d, int n_valid,
                                  int* flag_count, int* flag_list, int* list_cnt) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= m || n_valid <= kc) return;                // every valid row was re-scored
  const float s = screened[(long long)row * kc + kc - 1], e_k = out_dist[(long long)row * k + k - 1];
  const float2 qe = q_err[row];
  const float bound = d1_screen_bound(q_sq[row], qe.x, qe.y, db_max3[2], db_max3[0], db_max3[1], d, 3);
  if (!(s - bound > e_k)) {                             // also catches NaN
    const int f = atomicAdd(flag_count, 1);
    flag_list[f] = row;
    list_cnt[f] = 0;
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
  off[8] = take(dx_lists_at(m) + (size_t)m * DX_CAP * 8);   // list counters | lists of the exact fallback
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
  int* lcnt = reinterpret_cast<int*>(w + off[8]);
  unsigned long long* lists = reinterpret_cast<unsigned long long*>(w + off[8] + dx_lists_at(m));

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
    attr_done.mark();
  }
  const int sms = device_sm_count();
  gemm_f16_top16_kernel<<<g.total_items < sms ? g.total_items : sms, 160, D1_SMEM, s>>>(ma, mb, g);
  IBL_CUDA_OK(cudaGetLastError());

  FinishArgs f{};
  f.q = q; f.db = db; f.q_aux = qa; f.db_aux = da; f.db_max2 = dmax2; f.cand_d = cd; f.cand_i = ci;
  f.m = m; f.d = d; f.runs = g.items_per_mtile; f.k_out = k; f.n_valid = n_valid; f.idx_base = idx_base;
  f.out_dist = out_dist; f.out_idx = out_idx; f.flag_count = fcount; f.flag_list = flist; f.list_cnt = lcnt;
  const size_t qsm = d <= 16384 ? (size_t)d * sizeof(float) : 16;
  dist_finish_kernel<<<m, 128, qsm, s>>>(f);
  IBL_CUDA_OK(cudaGetLastError());

  ExactArgs x{};
  x.q = q; x.db = db; x.q_sq = reinterpret_cast<const float*>(qa); x.db_sq = reinterpret_cast<const float*>(da);
  x.sq_stride = 4; x.m = m; x.d = d; x.n_valid = n_valid; x.k = k;
  x.idx_base = idx_base; x.flag_count = fcount; x.flag_list = flist; x.list_cnt = lcnt; x.lists = lists;
  x.out_dist = out_dist; x.out_idx = out_idx;
  IBL_RET(dx_scan_attr());
  dist_exact_scan_kernel<<<device_sm_count(), DX_SCAN_WARPS * 32, dx_scan_smem(d), s>>>(x);   // exits at once when nothing is listed
  dist_exact_finish_kernel<<<64, 256, 0, s>>>(x);
  IBL_CUDA_OK(cudaGetLastError());
  if (launches) *launches += 7;
  return IBL_OK;
}

// the guard's counter of listed queries in this workspace (test hook ibl_debug_dist_flagged)
const int* dist1_flag_counter(const void* ws, int m, int n, int d) {
  size_t off[9];
  dist1_workspace_bytes(m, n, d, off);
  return reinterpret_cast<const int*>(reinterpret_cast<const uint8_t*>(ws) + off[4] + 16);
}

// layout: flag count, database maxima (256 B) | flag list [m], list counters [m] | lists [m][DX_CAP] keys
static size_t guard_lists_at(int m) { return 256 + (((size_t)m * 8 + 255) & ~(size_t)255); }
size_t dist_guard_workspace_bytes(int m) { return guard_lists_at(m) + (size_t)m * DX_CAP * 8; }

// Guard + exact fallback after a bf16x3 screening pass and its exact re-scoring (out_dist / out_idx hold the
// re-scored top-k).  screened [m][kc]: the kc candidates' screened distances, ascending.  q_err / db_err per row:
// {|lo|, |x - hi - lo|} (planes_sqnorm_kernel).  ws: dist_guard_workspace_bytes(m); its first int
// counts the listed queries.
int launch_dist_guard_bf16x3(const float* q, const float* q_sq, const float2* q_err, int m, const float* db,
                             const float* db_sq, const float2* db_err, int n_valid, int d, const float* screened, int kc,
                             int k, long long idx_base, void* ws, float* out_dist, long long* out_idx,
                             uint64_t* launches, cudaStream_t s) {
  IBL_REQUIRE(n_valid >= 1 && k >= 1 && k <= 128 && kc >= k, "bf16x3 guard: 1 <= k <= kc, k <= 128");
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  int* fcount = reinterpret_cast<int*>(w);
  float* dmax3 = reinterpret_cast<float*>(w + 16);
  int* flist = reinterpret_cast<int*>(w + 256);
  int* lcnt = flist + m;
  unsigned long long* lists = reinterpret_cast<unsigned long long*>(w + guard_lists_at(m));
  IBL_CUDA_OK(cudaMemsetAsync(w, 0, 32, s));
  dist_guard_colmax_kernel<<<cdiv(n_valid, 256) < 64 ? cdiv(n_valid, 256) : 64, 256, 0, s>>>(db_err, db_sq, n_valid, dmax3);
  dist_guard_kernel<<<cdiv(m, 128), 128, 0, s>>>(screened, kc, q_sq, q_err, dmax3, out_dist, k, m, d, n_valid, fcount,
                                                flist, lcnt);
  ExactArgs x{};
  x.q = q; x.db = db; x.q_sq = q_sq; x.db_sq = db_sq; x.sq_stride = 1; x.m = m; x.d = d; x.n_valid = n_valid; x.k = k;
  x.idx_base = idx_base; x.flag_count = fcount; x.flag_list = flist; x.list_cnt = lcnt; x.lists = lists;
  x.out_dist = out_dist; x.out_idx = out_idx;
  IBL_RET(dx_scan_attr());
  dist_exact_scan_kernel<<<device_sm_count(), DX_SCAN_WARPS * 32, dx_scan_smem(d), s>>>(x);   // exits at once when nothing is listed
  dist_exact_finish_kernel<<<64, 256, 0, s>>>(x);
  IBL_CUDA_OK(cudaGetLastError());
  if (launches) *launches += 4;
  return IBL_OK;
}

}  // namespace ibl
