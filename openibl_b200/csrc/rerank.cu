// k-reciprocal re-ranking (Zhong et al., CVPR 2017) on sparse data, the function of the reference's
// ibl/utils/rerank.py:32-100 (Evaluator.evaluate(rerank=True), evaluators.py:194-199) without any [N,N] array.
//
// Two entry points (include/iblb200.h), so that the dense work can be split over ranks:
//   1. neighbour pass (launch_knn_rowmax): for a block of rows of X [N,d], the first w columns ascending by
//      (d^2, index) and the row maximum M = max_j d^2, every value an exact fp32 distance (d1_exact).  Screening runs
//      on the tensor cores (bf16x3 dense tiles, launch_dist_dense_tc) in 32768-column chunks; per chunk the nearest
//      kn = w + 8 screened columns (launch_topk_rows) and the KNN_FAR farthest (knn_far_select_kernel) are kept and
//      re-scored exactly.  Two guards with the screening bound B of dist_exact.cuh decide whether the re-scored lists
//      are provably the exact answer; rows they cannot clear are ranked again by an exact scan of all N columns.
//   2. sparse stage (launch_rerank_topk), one warp or block per row, the sets in shared memory:
//        Kr / Kc      k-reciprocal sets of width k1+1 and round(k1/2)+1                    (rerank.py:51-57,60-64)
//        E            Kr plus every Kc[c], c in Kr, with |Kc[c] n Kr| > 2/3 |Kc[c]|, sorted unique (rerank.py:58-68)
//        V (CSR)      exp(-d^2/M) on E over its sum (ascending columns)                     (rerank.py:69-70)
//        k2 mean      V rows of the first k2 neighbours, summed in list order, / k2        (rerank.py:71-76)
//        inverted index of the gallery rows: a stable device radix sort of (column, row, value)
//        Jaccard      per query, (row, contribution) pairs emitted in ascending column order and stably sorted by
//                     row, so t[i,r] = sum_j min(V[i,j], V[r,j]) is summed in ascending j like rerank.py:90-92
//        top-k        over the overlap rows plus the rows that can precede every other one: the first k_orig rows
//                     of the original ranking (lambda > 0) or the lowest-index rows without overlap (lambda = 0).
//      No floating-point sum depends on scheduling: results are bit-identical from run to run.
//   3. dense entry (launch_rerank_dense), the reference function's own call shape: q-g, q-q and g-g distance matrices
//      in, the full [m,n] final matrix out.  D = [[qq, qg], [qg^T, gg]]; the reference squares D, divides every COLUMN
//      by its maximum and transposes (rerank.py:41-42), so row i of its matrix is column i of D, q(i,j) = D[j][i]^2 / M_i
//      with M_i = max_r D[r][i]^2.  Every read below is D[j][i]: the q-q and g-g inputs need not be bitwise symmetric.
//        neighbour pass  dn_knn_kernel: per column of D, M_i and the first w rows ascending by (q, index)
//        sparse stage    as above, the expansion reading the distances it recomputes from D (rr_expand_kernel<1, true>)
//        output          every entry (1 - lambda) + lambda q, then the overlap pairs overwritten with their Jaccard term
#include <cub/cub.cuh>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "dist_exact.cuh"

namespace ibl {

// ------------------------------------------------------------------------------------------------------------------
// shared helpers
// ------------------------------------------------------------------------------------------------------------------

// ascending bitonic sort of n (power of two) u64 keys in shared memory, any block size
__device__ void rr_sort_u64(unsigned long long* buf, int n) {
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long a = buf[lo], b = buf[hi];
        if ((a > b) == up) { buf[lo] = b; buf[hi] = a; }
      }
    }
  }
  __syncthreads();
}

// key of (d^2, column): d^2 >= 0, so its bit pattern orders like the value
__device__ __forceinline__ unsigned long long sq_key(float e, unsigned col) {
  return ((unsigned long long)__float_as_uint(__fmul_rn(e, e)) << 32) | col;
}

static int pow2_at_least(long long v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

// ------------------------------------------------------------------------------------------------------------------
// 1. neighbour pass
// ------------------------------------------------------------------------------------------------------------------
constexpr int KNN_FAR = 8;          // farthest screened columns kept per row and column chunk
constexpr int KNN_CHT = 32768;      // columns per dense screening chunk
constexpr int KNN_ROWS = 1024;      // rows per dense screening chunk (128 MB of screened distances)

// max over the rows of {|lo|, |x - hi - lo|, |x|^2}: the column side of the bound B
__global__ void knn_colmax_kernel(const float2* __restrict__ err, const float* __restrict__ sq, int n,
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

// One block per row of a screened chunk [rows][ld], nc valid columns starting at global column j0.  Every thread
// keeps its two largest screened values; the KNN_FAR largest thread maxima are the row's far candidates, and
// u = max(the next thread maximum, every thread's second largest) bounds the screened value of every column that
// was not kept (-inf: every column was kept).
__global__ void __launch_bounds__(256)
knn_far_select_kernel(const float* __restrict__ chunk, long long ld, int nc, int j0, int rows,
                      float* __restrict__ far_s, int* __restrict__ far_i, float* __restrict__ far_u) {
  __shared__ unsigned long long keys[256];
  __shared__ float red[8];
  const long long row = blockIdx.x;
  const float* p = chunk + row * ld;
  float s1 = -INFINITY, s2 = -INFINITY;
  int i1 = -1;
  for (int j = threadIdx.x; j < nc; j += 256) {
    const float v = __ldg(p + j);
    if (i1 < 0 || v > s1) { s2 = s1; s1 = v; i1 = j; }
    else if (v > s2) s2 = v;
  }
  keys[threadIdx.x] = i1 < 0 ? ~0ull : ((unsigned long long)(~d1_ord(s1)) << 32) | (unsigned)i1;   // largest first
  float m2 = s2;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m2;
  rr_sort_u64(keys, 256);
  if (threadIdx.x < KNN_FAR) {
    const unsigned long long k = keys[threadIdx.x];
    far_s[row * KNN_FAR + threadIdx.x] = k == ~0ull ? -INFINITY : d1_unord(~(uint32_t)(k >> 32));
    far_i[row * KNN_FAR + threadIdx.x] = k == ~0ull ? -1 : j0 + (int)(uint32_t)(k & 0xffffffffu);
  }
  if (threadIdx.x == 0) {
    float u = -INFINITY;
    for (int i = 0; i < 8; ++i) u = fmaxf(u, red[i]);
    const unsigned long long k = keys[KNN_FAR];
    if (k != ~0ull) u = fmaxf(u, d1_unord(~(uint32_t)(k >> 32)));
    far_u[row] = u;
  }
  (void)rows;
}

struct KnnFinishArgs {
  const float* x; int N, d;            // X, row stride d (d % 64 == 0)
  const float* sq; const float2* err;  // exact |x|^2 and {|lo|, |x - hi - lo|} of every row
  const float* colmax3;                // max over the rows of {|lo|, |res|, |x|^2}
  int row0, R;                         // rows row0 .. row0 + R - 1 of X
  const float* near_s; const long long* near_i; int kn;            // [R][kn] screened, ascending
  const float* far_s; const int* far_i; const float* far_u; int nch;   // [nch][R][KNN_FAR], [nch][R]
  int w;
  long long* out_idx; float* out_dist; float* out_max;             // [R][w], [R][w], [R]
  int* flag_count; int* flag_list;
  int* flag_total;                     // rows listed over the whole call (ibl_debug_knn_flagged)
};

// one block of 128 threads per row: exact re-scoring of the near and far candidates, sort by (d^2, index), guards
__global__ void __launch_bounds__(128)
knn_finish_kernel(const KnnFinishArgs g) {
  __shared__ unsigned long long keys[256];
  __shared__ float ex[256];
  __shared__ float wmax[4];
  const int row = blockIdx.x;
  const long long grow = g.row0 + row;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* xr = g.x + grow * g.d;
  const float an = __ldg(g.sq + grow);
  float mx = 0.f;
  for (int c = wid; c < 256; c += 4) {
    unsigned long long key = ~0ull;
    float e = 0.f;
    if (c < g.kn) {
      const long long ci = g.near_i[(long long)row * g.kn + c];
      if (ci >= 0) {
        e = d1_exact(xr, g.x + ci * g.d, g.d, lane, an, __ldg(g.sq + ci));
        key = sq_key(e, (unsigned)ci);
        mx = fmaxf(mx, __fmul_rn(e, e));
      }
    }
    if (lane == 0) { keys[c] = key; ex[c] = e; }
  }
  for (int c = wid; c < g.nch * KNN_FAR; c += 4) {
    const int ch = c / KNN_FAR, t = c - ch * KNN_FAR;
    const int ci = g.far_i[((long long)ch * g.R + row) * KNN_FAR + t];
    if (ci >= 0) {
      const float e = d1_exact(xr, g.x + (long long)ci * g.d, g.d, lane, an, __ldg(g.sq + ci));
      mx = fmaxf(mx, __fmul_rn(e, e));
    }
  }
  if (lane == 0) wmax[wid] = mx;
  __syncthreads();
  const float emax2 = fmaxf(fmaxf(wmax[0], wmax[1]), fmaxf(wmax[2], wmax[3]));
  // keys[c] is tied to ex[c] through the column; sort a copy of the keys only and look the distance up
  __shared__ unsigned long long sk[256];
  for (int i = threadIdx.x; i < 256; i += 128) sk[i] = keys[i];
  rr_sort_u64(sk, 256);
  for (int t = threadIdx.x; t < g.w; t += 128) {
    const unsigned long long k = sk[t];
    float e = INFINITY;
    long long idx = -1;
    if (k != ~0ull) {
      for (int c = 0; c < g.kn; ++c)
        if (keys[c] == k) { e = ex[c]; break; }
      idx = (long long)(uint32_t)(k & 0xffffffffu);
    }
    g.out_idx[(long long)row * g.w + t] = idx;
    g.out_dist[(long long)row * g.w + t] = e;
  }
  if (threadIdx.x == 0) {
    g.out_max[row] = emax2;
    const float2 qe = __ldg(g.err + grow);
    const double B = (double)d1_screen_bound(an, qe.x, qe.y, __ldg(g.colmax3 + 2), __ldg(g.colmax3), __ldg(g.colmax3 + 1),
                                             g.d, 3);
    bool ok = true;
    // near list: a column that was not kept has screened distance >= s_kn, so exact distance >= L = s_kn - B; it
    // cannot enter the first w when L > 0 and L^2 exceeds the w-th kept d^2
    if (g.N > g.kn) {
      const float skn = g.near_s[(long long)row * g.kn + g.kn - 1];
      const unsigned long long kw = sk[g.w - 1];
      const double L = (double)skn - B;
      ok = kw != ~0ull && L > 0.0 && L * L > (double)__uint_as_float((uint32_t)(kw >> 32)) * (1.0 + 1e-6);
    }
    // row maximum: a column in no far list has screened value <= u (max over the chunks) and >= the row's smallest
    // screened value, so its exact d^2 is at most max((u + B)^2, (B - s_min)^2)
    float u = -INFINITY;
    for (int c = 0; c < g.nch; ++c) u = fmaxf(u, g.far_u[(long long)c * g.R + row]);
    if (ok && u > -INFINITY) {
      const double hi = fmax((double)u + B, 0.0), lo = fmax(B - (double)g.near_s[(long long)row * g.kn], 0.0);
      ok = fmax(hi * hi, lo * lo) * (1.0 + 1e-6) < (double)emax2;
    }
    if (!ok) g.flag_list[atomicAdd(g.flag_count, 1)] = row;
  }
}

// Rows the guards could not clear: an exact scan of all N columns, 256 at a time, keeping the best 256 (d^2, index)
// keys and the maximum.  One block per listed row.
__global__ void __launch_bounds__(256)
knn_exact_kernel(const KnnFinishArgs g) {
  __shared__ unsigned long long keys[512];
  __shared__ float wmax[8];
  const int count = *g.flag_count;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (blockIdx.x == 0 && threadIdx.x == 0 && count > 0) atomicAdd(g.flag_total, count);
  for (int f = blockIdx.x; f < count; f += gridDim.x) {
    const int row = g.flag_list[f];
    const long long grow = g.row0 + row;
    const float* xr = g.x + grow * g.d;
    const float an = __ldg(g.sq + grow);
    __syncthreads();
    keys[threadIdx.x] = ~0ull;                // the best-so-far half; every scan step writes all of keys[256, 512)
    float mx = 0.f;
    for (int j0 = 0; j0 < g.N; j0 += 256) {
      for (int t = wid; t < 256; t += 8) {
        const int j = j0 + t;
        unsigned long long key = ~0ull;
        if (j < g.N) {
          const float e = d1_exact(xr, g.x + (long long)j * g.d, g.d, lane, an, __ldg(g.sq + j));
          key = sq_key(e, (unsigned)j);
          mx = fmaxf(mx, __fmul_rn(e, e));
        }
        if (lane == 0) keys[256 + t] = key;
      }
      rr_sort_u64(keys, 512);
    }
    if (lane == 0) wmax[wid] = mx;
    for (int t = wid; t < g.w; t += 8) {      // the signed distance of each listed column, recomputed
      const unsigned long long k = keys[t];
      float e = INFINITY;
      long long idx = -1;
      if (k != ~0ull) {
        idx = (long long)(uint32_t)(k & 0xffffffffu);
        e = d1_exact(xr, g.x + idx * g.d, g.d, lane, an, __ldg(g.sq + idx));
      }
      if (lane == 0) {
        g.out_idx[(long long)row * g.w + t] = idx;
        g.out_dist[(long long)row * g.w + t] = e;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float m = 0.f;
      for (int i = 0; i < 8; ++i) m = fmaxf(m, wmax[i]);
      g.out_max[row] = m;
    }
  }
}

struct KnnLayout {
  size_t off[13];
  size_t total;
  int dp, R, chw, nch, kn;
};

static KnnLayout knn_layout(int N, int d, int n_rows, int w) {
  KnnLayout L{};
  L.dp = (d + 63) / 64 * 64;
  L.R = n_rows < KNN_ROWS ? n_rows : KNN_ROWS;
  L.chw = N < KNN_CHT ? cdiv(N, 4) * 4 : KNN_CHT;
  L.nch = cdiv(N, KNN_CHT);
  L.kn = w + 8;
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += (bytes + 255) & ~(size_t)255; return at; };
  L.off[0] = take(L.dp == d ? 0 : (size_t)N * L.dp * 4);          // X padded to d % 64 == 0
  L.off[1] = take((size_t)N * L.dp * 4);                           // bf16 hi | lo planes
  L.off[2] = take((size_t)N * 4);                                  // |x|^2
  L.off[3] = take((size_t)N * 8);                                  // {|lo|, |res|}
  L.off[4] = take(256);                                            // column maxima, flag count
  L.off[5] = take((size_t)L.R * L.chw * 4);                        // screened chunk
  L.off[6] = take((size_t)L.nch * L.R * L.kn * 4);                 // near candidates per chunk
  L.off[7] = take((size_t)L.nch * L.R * L.kn * 8);
  L.off[8] = take((size_t)L.R * L.kn * 4);                         // merged near candidates: distances
  L.off[9] = take((size_t)L.nch * L.R * KNN_FAR * 8);              // far candidates (dist | idx)
  L.off[10] = take((size_t)L.nch * L.R * 4);                       // far bounds
  L.off[11] = take((size_t)L.R * 4);                               // flag list
  L.off[12] = take((size_t)L.R * L.kn * 8);                        // merged near candidates: int64 indices
  L.total = o;
  return L;
}

size_t knn_rowmax_workspace_bytes(int N, int d, int n_rows, int w) { return knn_layout(N, d, n_rows, w).total; }

// rows the guards sent to the exact scan in the last launch_knn_rowmax on this workspace
const int* knn_rowmax_flag_counter(const void* ws, int N, int d, int n_rows, int w) {
  return reinterpret_cast<const int*>(reinterpret_cast<const uint8_t*>(ws) + knn_layout(N, d, n_rows, w).off[4] + 20);
}

int launch_knn_rowmax(const float* X, int N, int d, int row0, int n_rows, int w, void* ws, long long* out_idx,
                      float* out_dist, float* out_max, uint64_t* launches, cudaStream_t s) {
  IBL_REQUIRE(w >= 1 && w <= 128 && w <= N, "knn_rowmax: 1 <= w <= min(128, N)");
  if (n_rows == 0) return IBL_OK;
  const KnnLayout L = knn_layout(N, d, n_rows, w);
  uint8_t* b = reinterpret_cast<uint8_t*>(ws);
  const int dp = L.dp;
  const float* x = X;
  if (dp != d) {                                   // zero columns change no product and no exact distance
    float* xp = reinterpret_cast<float*>(b + L.off[0]);
    IBL_CUDA_OK(cudaMemsetAsync(xp, 0, (size_t)N * dp * 4, s));
    IBL_CUDA_OK(cudaMemcpy2DAsync(xp, (size_t)dp * 4, X, (size_t)d * 4, (size_t)d * 4, N, cudaMemcpyDeviceToDevice, s));
    x = xp;
  }
  const size_t ne = (size_t)N * dp;
  __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(b + L.off[1]);
  __nv_bfloat16* lo = hi + ne;
  float* sq = reinterpret_cast<float*>(b + L.off[2]);
  float2* err = reinterpret_cast<float2*>(b + L.off[3]);
  float* cmax = reinterpret_cast<float*>(b + L.off[4]);
  int* fcount = reinterpret_cast<int*>(b + L.off[4] + 16);
  int* ftotal = fcount + 1;
  float* chunk = reinterpret_cast<float*>(b + L.off[5]);
  float* cd = reinterpret_cast<float*>(b + L.off[6]);
  int64_t* ci = reinterpret_cast<int64_t*>(b + L.off[7]);
  float* md = reinterpret_cast<float*>(b + L.off[8]);
  int64_t* mi = reinterpret_cast<int64_t*>(b + L.off[12]);
  float* fs = reinterpret_cast<float*>(b + L.off[9]);
  int* fi = reinterpret_cast<int*>(b + L.off[9] + (size_t)L.nch * L.R * KNN_FAR * 4);
  float* fu = reinterpret_cast<float*>(b + L.off[10]);
  int* flist = reinterpret_cast<int*>(b + L.off[11]);

  IBL_RET(launch_planes_sqnorm(x, N, dp, hi, lo, sq, err, s));
  IBL_CUDA_OK(cudaMemsetAsync(cmax, 0, 32, s));   // column maxima, this chunk's and the call's listed rows
  knn_colmax_kernel<<<std::min(64, cdiv(N, 256)), 256, 0, s>>>(err, sq, N, cmax);
  IBL_CUDA_OK(cudaGetLastError());
  uint64_t nl = 3;
  const int kn = std::min(L.kn, N);                // near candidates per row (all columns when N <= w + 8)
  for (int r0 = 0; r0 < n_rows; r0 += L.R) {
    const int R = std::min(L.R, n_rows - r0);
    const long long g0 = (long long)row0 + r0;
    IBL_CUDA_OK(cudaMemsetAsync(fcount, 0, 4, s));
    for (int c = 0; c < L.nch; ++c) {
      const int j0 = c * KNN_CHT, nc = std::min(KNN_CHT, N - j0);
      IBL_RET(launch_dist_dense_tc(hi + g0 * dp, lo + g0 * dp, sq + g0, R, hi + (size_t)j0 * dp, lo + (size_t)j0 * dp,
                                   sq + j0, nc, dp, chunk, L.chw, s));
      IBL_RET(launch_topk_rows(chunk, L.chw, R, nc, kn, j0, cd + (size_t)c * R * kn, ci + (size_t)c * R * kn, false,
                               s));
      knn_far_select_kernel<<<R, 256, 0, s>>>(chunk, L.chw, nc, j0, R, fs + (size_t)c * R * KNN_FAR,
                                              fi + (size_t)c * R * KNN_FAR, fu + (size_t)c * R);
      IBL_CUDA_OK(cudaGetLastError());
      nl += 3;
    }
    if (L.nch > 1) {
      IBL_RET(launch_topk_merge(cd, ci, L.nch, R, kn, kn, md, mi, s));
      ++nl;
    } else {
      md = cd;
      mi = ci;
    }
    KnnFinishArgs f{};
    f.x = x; f.N = N; f.d = dp; f.sq = sq; f.err = err; f.colmax3 = cmax; f.row0 = (int)g0; f.R = R;
    f.near_s = md; f.near_i = reinterpret_cast<const long long*>(mi); f.kn = kn;
    f.far_s = fs; f.far_i = fi; f.far_u = fu; f.nch = L.nch; f.w = w;
    f.out_idx = out_idx + (size_t)r0 * w; f.out_dist = out_dist + (size_t)r0 * w; f.out_max = out_max + r0;
    f.flag_count = fcount; f.flag_list = flist; f.flag_total = ftotal;
    knn_finish_kernel<<<R, 128, 0, s>>>(f);
    knn_exact_kernel<<<std::min(R, 4 * device_sm_count()), 256, 0, s>>>(f);   // exits at once when nothing is listed
    IBL_CUDA_OK(cudaGetLastError());
    nl += 2;
  }
  if (launches) *launches += nl;
  return IBL_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// 1b. neighbour pass over dense distance matrices (launch_rerank_dense)
// ------------------------------------------------------------------------------------------------------------------

// D = [[qq, qg], [qg^T, gg]] of m queries and n gallery rows, every input row-major fp32
struct DenseSrc {
  const float* qg; const float* qq; const float* gg;
  int m, n;
};

// D[r][c]
__device__ __forceinline__ float dense_at(const DenseSrc& s, long long r, long long c) {
  if (r < s.m) return c < s.m ? s.qq[r * s.m + c] : s.qg[r * s.n + (c - s.m)];
  return c < s.m ? s.qg[c * s.n + (r - s.m)] : s.gg[(r - s.m) * s.n + (c - s.m)];
}

constexpr int DN_WARPS = 4;          // row slices per block of 32 columns

// tile[k][l] = D[r0 + k][c0 + l] for the entries inside D.  Every input is read along its rows: the qg^T block (rows
// >= m, columns < m) as rows of qg, stored transposed.
__device__ __forceinline__ void dn_load_tile(const DenseSrc& s, int N, int r0, int c0, int lane, float (*tile)[33]) {
  __syncwarp();
  if (!(r0 >= s.m && c0 + 31 < s.m)) {
#pragma unroll 4
    for (int k = 0; k < 32; ++k) {
      const int r = r0 + k, c = c0 + lane;
      if (r < N && c < N && !(r >= s.m && c < s.m)) tile[k][lane] = dense_at(s, r, c);
    }
  }
  if (r0 + 31 >= s.m && c0 < s.m) {
#pragma unroll 4
    for (int k = 0; k < 32; ++k) {
      const int r = r0 + lane, c = c0 + k;
      if (r < N && c < N && r >= s.m && c < s.m) tile[lane][k] = dense_at(s, r, c);
    }
  }
  __syncwarp();
}

// One block of DN_WARPS warps per 32 columns c0 .. c0+31 of D (rows of the reference's matrix), lane l on column
// c0 + l; warp v streams down the 32-row tiles v, v + DN_WARPS, ...
//   sweep 1: M_c = max_r fl(D[r][c]^2)
//   sweep 2: keys (bits of q = fl(D[r][c]^2) / M_c, r), the slice's first w kept sorted in shared memory.  q >= 0, so
//            its bits order like the value; a later row never displaces an equal q, as in a stable sort.
// The DN_WARPS slices are merged per column -> idx [N,w], D[idx][c] [N,w], M [N]: the layout of launch_knn_rowmax.
__global__ void __launch_bounds__(DN_WARPS * 32)
dn_knn_kernel(const DenseSrc s, int w, long long* __restrict__ out_idx, float* __restrict__ out_dist,
              float* __restrict__ out_max) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned long long* lst = reinterpret_cast<unsigned long long*>(smem);                 // [DN_WARPS][w][32]
  float(*tiles)[32][33] = reinterpret_cast<float(*)[32][33]>(lst + (size_t)DN_WARPS * w * 32);
  __shared__ float wmax[DN_WARPS][32];
  const int N = s.m + s.n;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 32;
  float(*tile)[33] = tiles[wid];
  float mx = 0.f;
  for (int r0 = wid * 32; r0 < N; r0 += DN_WARPS * 32) {
    dn_load_tile(s, N, r0, c0, lane, tile);
    const int nr = min(32, N - r0);
    for (int k = 0; k < nr; ++k) {
      const float v = tile[k][lane];
      mx = fmaxf(mx, __fmul_rn(v, v));
    }
  }
  wmax[wid][lane] = mx;
  unsigned long long* my = lst + (size_t)wid * w * 32 + lane;         // slot t at my[t * 32]
  for (int t = 0; t < w; ++t) my[t * 32] = ~0ull;
  __syncthreads();
  float M = wmax[0][lane];
#pragma unroll
  for (int v = 1; v < DN_WARPS; ++v) M = fmaxf(M, wmax[v][lane]);
  unsigned long long thr = ~0ull;                                      // the slice's w-th key
  for (int r0 = wid * 32; r0 < N; r0 += DN_WARPS * 32) {
    dn_load_tile(s, N, r0, c0, lane, tile);
    const int nr = min(32, N - r0);
#pragma unroll 1
    for (int k = 0; k < nr; ++k) {
      const float v = tile[k][lane];
      const unsigned long long key =
          ((unsigned long long)__float_as_uint(__fdiv_rn(__fmul_rn(v, v), M)) << 32) | (unsigned)(r0 + k);
      if (key < thr) {
        int p = w - 1;
        while (p > 0 && my[(p - 1) * 32] > key) {
          my[p * 32] = my[(p - 1) * 32];
          --p;
        }
        my[p * 32] = key;
        thr = my[(w - 1) * 32];
      }
    }
  }
  __syncthreads();
  const int c = c0 + lane;
  if (wid != 0 || c >= N) return;
  int h[DN_WARPS] = {};
  for (int t = 0; t < w; ++t) {
    unsigned long long best = ~0ull;
    int bv = 0;
#pragma unroll
    for (int v = 0; v < DN_WARPS; ++v) {
      const unsigned long long k = h[v] < w ? lst[((size_t)v * w + h[v]) * 32 + lane] : ~0ull;
      if (k < best) { best = k; bv = v; }
    }
#pragma unroll
    for (int v = 0; v < DN_WARPS; ++v) h[v] += (v == bv);
    const long long r = best == ~0ull ? -1 : (long long)(uint32_t)(best & 0xffffffffu);
    out_idx[(long long)c * w + t] = r;
    out_dist[(long long)c * w + t] = r < 0 ? INFINITY : dense_at(s, r, c);
  }
  out_max[c] = M;
}

static size_t dn_knn_smem(int w) { return (size_t)DN_WARPS * w * 32 * 8 + (size_t)DN_WARPS * 32 * 33 * 4; }

// ------------------------------------------------------------------------------------------------------------------
// 2. sparse stage
// ------------------------------------------------------------------------------------------------------------------

// reciprocal sets of width `width` (<= 128): S[i] = { j in R_i[:width] : i in R_j[:width] } in R_i's order.  One warp
// per row.
__global__ void rr_recip_kernel(const long long* __restrict__ nbr, int N, int w, int width, int* __restrict__ out,
                                int* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= N) return;
  int n = 0;
  for (int p0 = 0; p0 < width; p0 += 32) {
    const int p = p0 + lane;
    bool mutual = false;
    long long j = -1;
    if (p < width) {
      j = nbr[i * w + p];
      if (j >= 0)
        for (int t = 0; t < width; ++t)
          if (nbr[j * w + t] == i) { mutual = true; break; }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, mutual);
    if (mutual) out[i * width + n + __popc(bal & ((1u << lane) - 1u))] = (int)j;
    n += __popc(bal);
  }
  if (lane == 0) cnt[i] = n;
}

struct ExpandArgs {
  const float* x; int d; const float* sq;   // exact recompute of the distances that are not in the neighbour list
  const long long* nbr; const float* nbr_dist; int w; const float* rowmax;
  const int* kr; const int* kr_cnt; int wr;    // [N][wr]
  const int* kc; const int* kc_cnt; int wc;    // [N][wc]
  int N, cap;                                  // cap: power of two >= wr * (wc + 1)
  int* nnz;                                    // pass 0: [N] sizes
  const long long* rowptr; int* cols; float* vals;   // pass 1
  DenseSrc dn;                                 // DENSE: the distances are read from D instead (x, d, sq unused)
};

// E_i and V_i for one row per block (128 threads).  pass 0 counts |E_i|, pass 1 writes the CSR row.  A distance that
// is not in the neighbour list comes from the descriptors (d1_exact) or, DENSE, from D[j][i].
template <int PASS, bool DENSE = false>
__global__ void __launch_bounds__(128)
rr_expand_kernel(const ExpandArgs g) {
  extern __shared__ __align__(16) unsigned char smem[];
  int* buf = reinterpret_cast<int*>(smem);                        // [cap]
  float* val = reinterpret_cast<float*>(buf + g.cap);             // [cap]
  int* kr = reinterpret_cast<int*>(val + g.cap);                  // [wr]
  __shared__ int n_s, u_s;
  __shared__ float sum_s;
  const int i = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nr = g.kr_cnt[i];
  for (int t = threadIdx.x; t < nr; t += 128) { kr[t] = g.kr[(long long)i * g.wr + t]; buf[t] = kr[t]; }
  for (int t = nr + threadIdx.x; t < g.cap; t += 128) buf[t] = 0x7fffffff;
  if (threadIdx.x == 0) n_s = nr;
  __syncthreads();
  for (int a = wid; a < nr; a += 4) {
    const int c = kr[a];
    const int nc = g.kc_cnt[c];
    int inter = 0;
    for (int t0 = 0; t0 < nc; t0 += 32) {
      bool in = false;
      if (t0 + lane < nc) {
        const int v = g.kc[(long long)c * g.wc + t0 + lane];
        for (int q = 0; q < nr; ++q) in |= (kr[q] == v);
      }
      inter += __popc(__ballot_sync(0xffffffffu, in));
    }
    if ((double)inter > (2.0 / 3.0) * (double)nc) {          // rerank.py:65, in the reference's double arithmetic
      int at = 0;
      if (lane == 0) at = atomicAdd(&n_s, nc);
      at = __shfl_sync(0xffffffffu, at, 0);
      for (int t = lane; t < nc; t += 32) buf[at + t] = g.kc[(long long)c * g.wc + t];
    }
  }
  // bitonic sort of the int buffer
  for (int size = 2; size <= g.cap; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < (g.cap >> 1); t += 128) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const int a = buf[lo], b = buf[hi];
        if ((a > b) == up) { buf[lo] = b; buf[hi] = a; }
      }
    }
  }
  __syncthreads();
  // unique, in place (one thread: at most cap entries)
  if (threadIdx.x == 0) {
    int u = 0;
    for (int t = 0; t < g.cap && buf[t] != 0x7fffffff; ++t)
      if (u == 0 || buf[u - 1] != buf[t]) buf[u++] = buf[t];
    u_s = u;
  }
  __syncthreads();
  const int u = u_s;
  if (PASS == 0) {
    if (threadIdx.x == 0) g.nnz[i] = u;
    return;
  } else {
    // exp(-d^2 / M_i): the listed distance when the column is in the neighbour list, else an exact recompute
    const float M = g.rowmax[i];
    const float* xr = g.x + (long long)i * g.d;
    const float an = __ldg(g.sq + i);
    for (int t = wid; t < u; t += 4) {
      const int j = buf[t];
      float e = 0.f;
      bool found = false;
      for (int q0 = 0; q0 < g.w; q0 += 32) {
        const bool hit = (q0 + lane < g.w) && g.nbr[(long long)i * g.w + q0 + lane] == j;
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (bal) { e = g.nbr_dist[(long long)i * g.w + q0 + __ffs(bal) - 1]; found = true; break; }
      }
      if (!found) {
        if constexpr (DENSE) e = dense_at(g.dn, j, i);
        else e = d1_exact(xr, g.x + (long long)j * g.d, g.d, lane, an, __ldg(g.sq + j));
      }
      if (lane == 0) val[t] = expf(-__fdiv_rn(__fmul_rn(e, e), M));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
      for (int t = 0; t < u; ++t) s = __fadd_rn(s, val[t]);      // ascending column order
      sum_s = s;
    }
    __syncthreads();
    const long long o = g.rowptr[i];
    for (int t = threadIdx.x; t < u; t += 128) {
      g.cols[o + t] = buf[t];
      g.vals[o + t] = __fdiv_rn(val[t], sum_s);
    }
  }
}

struct MeanArgs {
  const long long* nbr; int w, k2;
  const long long* rowptr; const int* cols; const float* vals;   // V
  int cap;                                                       // power of two >= k2 * max row size
  int* nnz;                                                      // pass 0
  const long long* rowptr2; int* cols2; float* vals2;            // pass 1
};

// V'_i = mean of the V rows of i's first k2 neighbours (rerank.py:71-76): entries keyed (column, neighbour slot,
// position), sorted, each column summed in neighbour order and divided by k2.  One row per block (256 threads).
template <int PASS>
__global__ void __launch_bounds__(256)
rr_mean_kernel(const MeanArgs g) {
  extern __shared__ __align__(16) unsigned long long keys[];     // [cap]
  __shared__ int u_s;
  const long long i = blockIdx.x;
  __shared__ long long start[128];
  __shared__ int len[128];
  if (threadIdx.x < g.k2) {
    const long long q = g.nbr[i * g.w + threadIdx.x];
    start[threadIdx.x] = g.rowptr[q];
    len[threadIdx.x] = (int)(g.rowptr[q + 1] - g.rowptr[q]);
  }
  for (int t = threadIdx.x; t < g.cap; t += 256) keys[t] = ~0ull;
  __syncthreads();
  int base = 0;
  for (int q = 0; q < g.k2; ++q) {
    for (int t = threadIdx.x; t < len[q]; t += 256)
      keys[base + t] = ((unsigned long long)(unsigned)g.cols[start[q] + t] << 32) | ((unsigned)q << 24) | (unsigned)t;
    base += len[q];
  }
  rr_sort_u64(keys, g.cap);
  if (threadIdx.x == 0) {          // compact: one sum per column, in neighbour order
    int u = 0;
    const float fk2 = (float)g.k2;
    for (int t = 0; t < base; ) {
      const unsigned col = (unsigned)(keys[t] >> 32);
      float s = 0.f;
      int e = t;
      while (e < base && (unsigned)(keys[e] >> 32) == col) {
        if (PASS == 1) {
          const int q = (int)((keys[e] >> 24) & 0xff), pos = (int)(keys[e] & 0xffffff);
          s = __fadd_rn(s, g.vals[start[q] + pos]);
        }
        ++e;
      }
      if (PASS == 1) {
        g.cols2[g.rowptr2[i] + u] = (int)col;
        g.vals2[g.rowptr2[i] + u] = __fdiv_rn(s, fk2);
      }
      ++u;
      t = e;
    }
    u_s = u;
    if (PASS == 0) g.nnz[i] = u;
  }
}

// inverted index input: for gallery rows r >= m, (column, (r - m) << 32 | value bits), one warp per row
__global__ void rr_invert_emit_kernel(const long long* __restrict__ rowptr, const int* __restrict__ cols,
                                      const float* __restrict__ vals, int m, int N, unsigned* __restrict__ kcol,
                                      unsigned long long* __restrict__ vrow) {
  const int lane = threadIdx.x & 31;
  const long long r = m + (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= N) return;
  const long long b0 = rowptr[m];
  for (long long p = rowptr[r] + lane; p < rowptr[r + 1]; p += 32) {
    kcol[p - b0] = (unsigned)cols[p];
    vrow[p - b0] = ((unsigned long long)(r - m) << 32) | __float_as_uint(vals[p]);
  }
}

// colptr[j] = first position of column j in the sorted column keys (lower bound)
__global__ void rr_colptr_kernel(const unsigned* __restrict__ kcol, long long G, int N, long long* __restrict__ colptr) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j > N) return;
  long long lo = 0, hi = G;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if ((long long)kcol[mid] < j) lo = mid + 1; else hi = mid;
  }
  colptr[j] = lo;
}

// per query: the number of (gallery row, column) pairs it meets through its support
__global__ void rr_query_count_kernel(const long long* __restrict__ rowptr, const int* __restrict__ cols,
                                      const long long* __restrict__ colptr, int m, long long* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= m) return;
  long long c = 0;
  for (long long p = rowptr[i] + lane; p < rowptr[i + 1]; p += 32) {
    const int j = cols[p];
    c += colptr[j + 1] - colptr[j];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) out[i] = c;
}

// per query of a chunk, one warp: (query, gallery row) keys and min(V[i,j], V[r,j]), columns j in ascending order
__global__ void rr_pairs_emit_kernel(const long long* __restrict__ rowptr, const int* __restrict__ cols,
                                     const float* __restrict__ vals, const long long* __restrict__ colptr,
                                     const unsigned long long* __restrict__ vrow, const long long* __restrict__ qoff,
                                     int q0, int q1, long long base, long long n_gal,
                                     unsigned long long* __restrict__ keys, float* __restrict__ contrib) {
  const int lane = threadIdx.x & 31;
  const long long i = q0 + (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= q1) return;
  long long o = qoff[i] - base;
  const unsigned long long kq = (unsigned long long)(i - q0) * (unsigned long long)n_gal;
  for (long long p = rowptr[i]; p < rowptr[i + 1]; ++p) {
    const int j = cols[p];
    const float vi = vals[p];
    const long long c0 = colptr[j], c1 = colptr[j + 1];
    for (long long c = c0 + lane; c < c1; c += 32) {
      const unsigned long long e = vrow[c];
      keys[o + (c - c0)] = kq + (e >> 32);
      contrib[o + (c - c0)] = fminf(vi, __uint_as_float((uint32_t)(e & 0xffffffffu)));
    }
    o += c1 - c0;
  }
}

// t at the first position of every (query, row) run of the stably sorted pairs, summed in emission order
__global__ void rr_segment_sum_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ contrib,
                                      long long T, float* __restrict__ t_out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= T) return;
  const unsigned long long k = keys[p];
  if (p > 0 && keys[p - 1] == k) { t_out[p] = -1.f; return; }
  float s = 0.f;
  for (long long e = p; e < T && keys[e] == k; ++e) s = __fadd_rn(s, contrib[e]);
  t_out[p] = s;
}

struct TopkArgs {
  const float* x; int d; const float* sq; const float* rowmax;
  int m; long long n_gal;
  const unsigned long long* keys; const float* t; const long long* qoff; long long base; int q0;
  const long long* orig; int k_orig;
  float lam, oml;
  int k;
  float* out_dist; long long* out_idx;
};

__device__ __forceinline__ float rr_final(float jac, float dn, float lam, float oml) {
  return lam == 0.f ? jac : __fadd_rn(__fmul_rn(jac, oml), __fmul_rn(dn, lam));   // rerank.py:97
}

// one block (256 threads) per query of the chunk: top-k of the overlap rows and the rows that may precede them
__global__ void __launch_bounds__(256)
rr_topk_kernel(const TopkArgs g) {
  __shared__ unsigned long long best[512];
  __shared__ int rr[256];
  __shared__ float jj[256];
  __shared__ int cnt_s;
  const int qi = g.q0 + blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long lo = g.qoff[qi] - g.base, hi = g.qoff[qi + 1] - g.base;
  const unsigned long long kq = (unsigned long long)blockIdx.x * (unsigned long long)g.n_gal;
  const float* xr = g.x + (long long)qi * g.d;
  const float an = __ldg(g.sq + qi), M = g.rowmax[qi];
  for (int t = threadIdx.x; t < 512; t += 256) best[t] = ~0ull;
  // rows of the candidate set are scored 256 at a time into best[256, 512): (jac, row) first, then, with lambda > 0,
  // d^2 / M by the exact routine (one warp per row)
  auto score_tile = [&]() {
    __syncthreads();
    const int n = cnt_s;
    for (int t = wid; t < n; t += 8) {
      const int r = rr[t];
      float dn = 0.f;
      if (g.lam != 0.f) {
        const float e = d1_exact(xr, g.x + (long long)(g.m + r) * g.d, g.d, lane, an, __ldg(g.sq + g.m + r));
        dn = __fdiv_rn(__fmul_rn(e, e), M);
      }
      if (lane == 0) best[256 + t] = ((unsigned long long)d1_ord(rr_final(jj[t], dn, g.lam, g.oml)) << 32) | (unsigned)r;
    }
    __syncthreads();
    rr_sort_u64(best, 512);
    for (int t = threadIdx.x; t < 256; t += 256) best[256 + t] = ~0ull;
    __syncthreads();
  };
  for (long long p0 = lo; p0 < hi; p0 += 256) {
    __syncthreads();
    if (threadIdx.x == 0) cnt_s = 0;
    __syncthreads();
    const long long p = p0 + threadIdx.x;
    if (p < hi && g.t[p] >= 0.f) {
      const float t = g.t[p];
      const int at = atomicAdd(&cnt_s, 1);       // slot order does not matter: the keys are sorted afterwards
      rr[at] = (int)(g.keys[p] - kq);
      jj[at] = __fsub_rn(1.f, __fdiv_rn(t, __fsub_rn(2.f, t)));   // rerank.py:93
    }
    score_tile();
  }
  // rows without overlap score jac = 1
  __syncthreads();
  if (threadIdx.x == 0) cnt_s = 0;
  __syncthreads();
  auto in_overlap = [&](long long r) {
    long long a = lo, b = hi;
    const unsigned long long key = kq + (unsigned long long)r;
    while (a < b) {
      const long long mid = (a + b) >> 1;
      if (g.keys[mid] < key) a = mid + 1; else b = mid;
    }
    return a < hi && g.keys[a] == key;
  };
  if (g.lam != 0.f) {
    // a row outside the overlap and outside the first k rows of the original ranking has k rows before it
    for (int t = threadIdx.x; t < g.k_orig; t += 256) {
      const long long r = g.orig[(long long)qi * g.k_orig + t];
      if (r >= 0 && r < g.n_gal && !in_overlap(r)) {
        const int at = atomicAdd(&cnt_s, 1);
        rr[at] = (int)r;
        jj[at] = 1.f;
      }
    }
  } else if (threadIdx.x == 0) {
    // lambda = 0: every row outside the overlap scores exactly 1, so the lowest indices come first
    long long p = lo;
    int c = 0;
    for (long long r = 0; r < g.n_gal && c < g.k; ++r) {
      while (p < hi && g.keys[p] < kq + (unsigned long long)r) ++p;
      if (p < hi && g.keys[p] == kq + (unsigned long long)r) continue;
      rr[c] = (int)r;
      jj[c] = 1.f;
      ++c;
    }
    cnt_s = c;
  }
  score_tile();
  for (int t = threadIdx.x; t < g.k; t += 256) {
    const unsigned long long key = best[t];
    g.out_dist[(long long)qi * g.k + t] = key == ~0ull ? INFINITY : d1_unord((uint32_t)(key >> 32));
    g.out_idx[(long long)qi * g.k + t] = key == ~0ull ? -1 : (long long)(uint32_t)(key & 0xffffffffu);
  }
}

// final = fl(fl(jac * c1) + fl(q * c2)), c1 = fp32(1 - lambda), c2 = fp32(lambda): rerank.py:94 in float32 (NEP 50).
// Separate roundings: a contracted FMA is one ulp off the reference.
__device__ __forceinline__ float rr_dense_final(float jac, float q, float c1, float c2) {
  return __fadd_rn(__fmul_rn(jac, c1), __fmul_rn(q, c2));
}

// every (query i, gallery j) with jac = 1, q = fl(qg[i][j]^2) / M_i (D[m+j][i] is qg[i][j])
__global__ void rr_dense_base_kernel(const float* __restrict__ qg, const float* __restrict__ rowmax, int m, int n,
                                     float c1, float c2, float* __restrict__ out) {
  const long long total = (long long)m * n;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(p / n);
    const float v = __ldg(qg + p);
    out[p] = rr_dense_final(1.f, __fdiv_rn(__fmul_rn(v, v), __ldg(rowmax + i)), c1, c2);
  }
}

// the overlap pairs of a query chunk: t at the first position of each (query, row) run (rr_segment_sum_kernel).  Each
// pair is written once, so the output does not depend on scheduling.
__global__ void rr_dense_scatter_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ t,
                                        long long T, int q0, long long n_gal, const float* __restrict__ qg,
                                        const float* __restrict__ rowmax, float c1, float c2, float* __restrict__ out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= T) return;
  const float tp = t[p];
  if (tp < 0.f) return;
  const unsigned long long k = keys[p];
  const long long i = q0 + (long long)(k / (unsigned long long)n_gal), r = (long long)(k % (unsigned long long)n_gal);
  const float jac = __fsub_rn(1.f, __fdiv_rn(tp, __fsub_rn(2.f, tp)));   // rerank.py:92
  const float v = qg[i * n_gal + r];
  out[i * n_gal + r] = rr_dense_final(jac, __fdiv_rn(__fmul_rn(v, v), rowmax[i]), c1, c2);
}

// |x|^2 in planes_sqnorm_kernel's summation order (gemm_simt.cu), so that a distance recomputed here is bit-identical
// to the neighbour pass's distance of the same pair
__global__ void __launch_bounds__(256)
rr_sqnorm_kernel(const float* __restrict__ x, int D, float* __restrict__ sq) {
  __shared__ float red[8];
  const long long r = blockIdx.x;
  const float4* p = reinterpret_cast<const float4*>(x + r * D);
  float ss = 0.f;
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) {
    const float4 v = __ldg(p + i);
    ss = fmaf(v.x, v.x, ss); ss = fmaf(v.y, v.y, ss); ss = fmaf(v.z, v.z, ss); ss = fmaf(v.w, v.w, ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
    sq[r] = tot;
  }
}

// ---- host -------------------------------------------------------------------------------------------------------

struct RrBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes) {
    if (bytes <= cap) return IBL_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    const cudaError_t e = cudaMalloc(&p, bytes < 256 ? 256 : bytes);
    if (e != cudaSuccess) {
      cudaGetLastError();
      set_last_error("re-ranking workspace cudaMalloc(" + std::to_string(bytes) + " B) failed: " + cudaGetErrorString(e));
      return IBL_ERR_OOM;
    }
    cap = bytes < 256 ? 256 : bytes;
    return IBL_OK;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct RerankWs {
  RrBuf sets, nnz, rowptr, cols, vals, cols2, vals2, inv_v2, colptr, qcnt, qoff, pk, pk2, pv,
      pv2, tsum, temp, xpad, sq, dmax,
      dn;   // launch_rerank_dense: neighbour lists, their distances and the row maxima
};

RerankWs* rerank_ws_create() { return new RerankWs(); }
void rerank_ws_destroy(RerankWs* w) {
  if (!w) return;
  RrBuf* all[] = {&w->sets, &w->nnz, &w->rowptr, &w->cols, &w->vals, &w->cols2, &w->vals2, &w->inv_v2, &w->colptr, &w->qcnt, &w->qoff, &w->pk, &w->pk2, &w->pv,
                  &w->pv2, &w->tsum, &w->temp, &w->xpad, &w->sq, &w->dmax, &w->dn};
  for (RrBuf* b : all)
    if (b->p) cudaFree(b->p);
  delete w;
}
size_t rerank_ws_bytes(const RerankWs* w) {
  const RrBuf* all[] = {&w->sets, &w->nnz, &w->rowptr, &w->cols, &w->vals, &w->cols2, &w->vals2, &w->inv_v2, &w->colptr, &w->qcnt, &w->qoff, &w->pk, &w->pk2, &w->pv,
                        &w->pv2, &w->tsum, &w->temp, &w->xpad, &w->sq, &w->dmax, &w->dn};
  size_t s = 0;
  for (const RrBuf* b : all) s += b->cap;
  return s;
}

static int half_round_even(int k1) {            // int(np.around(k1 / 2.)), rerank.py:60
  if (k1 % 2 == 0) return k1 / 2;
  const int f = k1 / 2;                          // k1 / 2 = f + 0.5
  return (f % 2 == 0) ? f : f + 1;
}

// CSR row pointers from row sizes: exclusive scan on the device, total and largest row copied to the host
static int csr_rows(RerankWs* W, const int* nnz, int N, RrBuf& rowptr, long long* total, int* maxrow, cudaStream_t s) {
  IBL_RET(rowptr.ensure((size_t)(N + 1) * 8));
  long long* rp = rowptr.as<long long>();
  IBL_CUDA_OK(cudaMemsetAsync(rp, 0, 8, s));
  size_t tb = 0, tb2 = 0;
  IBL_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, tb, nnz, rp + 1, N, s));
  IBL_CUDA_OK(cub::DeviceReduce::Max(nullptr, tb2, nnz, reinterpret_cast<int*>(rp), N, s));
  IBL_RET(W->temp.ensure(std::max(tb, tb2) + 256));
  IBL_RET(W->dmax.ensure(16));
  int* dmax = W->dmax.as<int>();
  IBL_CUDA_OK(cub::DeviceScan::InclusiveSum(W->temp.p, tb, nnz, rp + 1, N, s));
  IBL_CUDA_OK(cub::DeviceReduce::Max(W->temp.p, tb2, nnz, dmax, N, s));
  IBL_CUDA_OK(cudaMemcpyAsync(total, rp + N, 8, cudaMemcpyDeviceToHost, s));
  IBL_CUDA_OK(cudaMemcpyAsync(maxrow, dmax, 4, cudaMemcpyDeviceToHost, s));
  IBL_CUDA_OK(cudaStreamSynchronize(s));
  return IBL_OK;
}

// Shared-memory limits of the kernels a path launches, set once per device.  Each path sets only its own kernels:
// setting an attribute loads the kernel's module, which the other path need not pay for.
template <bool DENSE>
static int rr_set_attributes() {
  static DeviceOnce attr;
  if (attr.done()) return IBL_OK;
  IBL_CUDA_OK(cudaFuncSetAttribute(rr_expand_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  IBL_CUDA_OK(cudaFuncSetAttribute(rr_expand_kernel<1, DENSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  IBL_CUDA_OK(cudaFuncSetAttribute(rr_mean_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  IBL_CUDA_OK(cudaFuncSetAttribute(rr_mean_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  if (DENSE)
    IBL_CUDA_OK(cudaFuncSetAttribute(dn_knn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dn_knn_smem(128)));
  attr.mark();
  return IBL_OK;
}

// The sparse stage from the [N,w] lists and M of all rows (ea: the distance source, nbr, nbr_dist, w, rowmax) up to
// the Jaccard sums.  For every chunk [q0, q1) of queries, emit(q0, q1, base, T) runs with the T stably sorted
// (query - q0, row) keys in W->pk2, t at the first position of each run in W->tsum (-1 elsewhere) and the chunk's
// offsets qoff[q0..q1] - base in W->qoff.
template <bool DENSE, class Emit>
static int rerank_sparse(RerankWs* W, ExpandArgs ea, int N, int m, int k1, int k2, uint64_t& nl, cudaStream_t s,
                         Emit&& emit) {
  const int wr = k1 + 1, wc = half_round_even(k1) + 1;
  const long long n_gal = (long long)N - m;
  const long long* nbr = ea.nbr;
  const int w = ea.w;
  // k-reciprocal sets
  IBL_RET(W->sets.ensure((size_t)N * (wr + wc + 2) * 4));
  int* kr = W->sets.as<int>();
  int* kc = kr + (size_t)N * wr;
  int* krc = kc + (size_t)N * wc;
  int* kcc = krc + N;
  rr_recip_kernel<<<cdiv(N, 8), 256, 0, s>>>(nbr, N, w, wr, kr, krc);
  rr_recip_kernel<<<cdiv(N, 8), 256, 0, s>>>(nbr, N, w, wc, kc, kcc);
  IBL_CUDA_OK(cudaGetLastError());
  nl += 3;
  // expansion + V
  ea.kr = kr; ea.kr_cnt = krc; ea.wr = wr; ea.kc = kc; ea.kc_cnt = kcc; ea.wc = wc; ea.N = N;
  ea.cap = pow2_at_least((long long)wr * (wc + 1));
  const size_t esm = (size_t)ea.cap * 8 + (size_t)wr * 4;
  IBL_REQUIRE(esm <= 200 * 1024, "re-ranking: k1 too large for the expansion kernel's shared memory");
  IBL_RET(rr_set_attributes<DENSE>());
  IBL_RET(W->nnz.ensure((size_t)N * 4));
  ea.nnz = W->nnz.as<int>();
  rr_expand_kernel<0><<<N, 128, esm, s>>>(ea);
  IBL_CUDA_OK(cudaGetLastError());
  long long nnz = 0;
  int maxrow = 0;
  IBL_RET(csr_rows(W, W->nnz.as<int>(), N, W->rowptr, &nnz, &maxrow, s));
  IBL_RET(W->cols.ensure((size_t)nnz * 4));
  IBL_RET(W->vals.ensure((size_t)nnz * 4));
  ea.rowptr = W->rowptr.as<long long>(); ea.cols = W->cols.as<int>(); ea.vals = W->vals.as<float>();
  rr_expand_kernel<1, DENSE><<<N, 128, esm, s>>>(ea);
  IBL_CUDA_OK(cudaGetLastError());
  nl += 4;
  const long long* rowptr = W->rowptr.as<long long>();
  const int* cols = W->cols.as<int>();
  const float* vals = W->vals.as<float>();
  if (k2 > 1) {
    MeanArgs ma{};
    ma.nbr = nbr; ma.w = w; ma.k2 = k2; ma.rowptr = rowptr; ma.cols = cols; ma.vals = vals;
    ma.cap = pow2_at_least((long long)k2 * maxrow);
    IBL_REQUIRE((size_t)ma.cap * 8 <= 200 * 1024 && maxrow < (1 << 24),
                "re-ranking: k2 x (largest expansion set) too large for the k2 mean kernel's shared memory");
    ma.nnz = W->nnz.as<int>();
    rr_mean_kernel<0><<<N, 256, (size_t)ma.cap * 8, s>>>(ma);
    IBL_CUDA_OK(cudaGetLastError());
    // the second CSR needs its own row pointers: W->pk holds them (it is free until the Jaccard pass)
    long long nnz2 = 0;
    int max2 = 0;
    IBL_RET(csr_rows(W, W->nnz.as<int>(), N, W->pk, &nnz2, &max2, s));
    IBL_RET(W->cols2.ensure((size_t)nnz2 * 4));
    IBL_RET(W->vals2.ensure((size_t)nnz2 * 4));
    ma.rowptr2 = W->pk.as<long long>(); ma.cols2 = W->cols2.as<int>(); ma.vals2 = W->vals2.as<float>();
    rr_mean_kernel<1><<<N, 256, (size_t)ma.cap * 8, s>>>(ma);
    IBL_CUDA_OK(cudaGetLastError());
    nl += 4;
    IBL_RET(W->rowptr.ensure((size_t)(N + 1) * 8));
    IBL_CUDA_OK(cudaMemcpyAsync(W->rowptr.p, W->pk.p, (size_t)(N + 1) * 8, cudaMemcpyDeviceToDevice, s));
    rowptr = W->rowptr.as<long long>();
    cols = W->cols2.as<int>();
    vals = W->vals2.as<float>();
    nnz = nnz2;
  }
  // inverted index over the gallery rows
  long long hb[2];
  IBL_CUDA_OK(cudaMemcpyAsync(hb, rowptr + m, 8, cudaMemcpyDeviceToHost, s));
  IBL_CUDA_OK(cudaStreamSynchronize(s));
  const long long G = nnz - hb[0];
  // the sort's column keys and input values are dead once colptr is built: they live in the pair buffers
  IBL_RET(W->pk.ensure((size_t)G * 8));
  IBL_RET(W->pk2.ensure((size_t)G * 8));
  unsigned* inv_k = W->pk.as<unsigned>();
  unsigned* inv_k2 = W->pk2.as<unsigned>();
  IBL_RET(W->pv.ensure((size_t)G * 8));
  unsigned long long* inv_v = W->pv.as<unsigned long long>();
  IBL_RET(W->inv_v2.ensure((size_t)G * 8));
  IBL_RET(W->colptr.ensure((size_t)(N + 1) * 8));
  if (n_gal > 0) {
    rr_invert_emit_kernel<<<cdiv(n_gal, 8), 256, 0, s>>>(rowptr, cols, vals, m, N, inv_k,
                                                         inv_v);
    IBL_CUDA_OK(cudaGetLastError());
  }
  int col_bits = 1;
  while ((1ll << col_bits) < N) ++col_bits;
  {
    size_t tb = 0;
    IBL_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, tb, inv_k, inv_k2,
                                                inv_v, W->inv_v2.as<unsigned long long>(),
                                                G, 0, col_bits, s));
    IBL_RET(W->temp.ensure(tb + 256));
    IBL_CUDA_OK(cub::DeviceRadixSort::SortPairs(W->temp.p, tb, inv_k, inv_k2,
                                                inv_v, W->inv_v2.as<unsigned long long>(),
                                                G, 0, col_bits, s));
  }
  rr_colptr_kernel<<<cdiv(N + 1, 256), 256, 0, s>>>(inv_k2, G, N, W->colptr.as<long long>());
  // pairs per query, planned into chunks on the host
  IBL_RET(W->qcnt.ensure((size_t)m * 8));
  IBL_RET(W->qoff.ensure((size_t)(m + 1) * 8));
  rr_query_count_kernel<<<cdiv(m, 8), 256, 0, s>>>(rowptr, cols, W->colptr.as<long long>(), m, W->qcnt.as<long long>());
  IBL_CUDA_OK(cudaGetLastError());
  nl += 4;
  std::vector<long long> qc(m), qo(m + 1, 0);
  IBL_CUDA_OK(cudaMemcpyAsync(qc.data(), W->qcnt.p, (size_t)m * 8, cudaMemcpyDeviceToHost, s));
  IBL_CUDA_OK(cudaStreamSynchronize(s));
  for (int i = 0; i < m; ++i) qo[i + 1] = qo[i] + qc[i];
  IBL_CUDA_OK(cudaMemcpyAsync(W->qoff.p, qo.data(), (size_t)(m + 1) * 8, cudaMemcpyHostToDevice, s));
  const long long budget = 1ll << 22;            // pairs sorted at once (4M: ~100 MB with the sort's buffers)
  for (int q0 = 0; q0 < m;) {
    int q1 = q0 + 1;
    while (q1 < m && qo[q1 + 1] - qo[q0] <= budget && q1 - q0 < 65535) ++q1;
    const long long T = qo[q1] - qo[q0];
    IBL_RET(W->pk.ensure((size_t)std::max(T, 1ll) * 8));
    IBL_RET(W->pk2.ensure((size_t)std::max(T, 1ll) * 8));
    IBL_RET(W->pv.ensure((size_t)std::max(T, 1ll) * 4));
    IBL_RET(W->pv2.ensure((size_t)std::max(T, 1ll) * 4));
    IBL_RET(W->tsum.ensure((size_t)std::max(T, 1ll) * 4));
    if (T > 0) {
      rr_pairs_emit_kernel<<<cdiv(q1 - q0, 8), 256, 0, s>>>(rowptr, cols, vals, W->colptr.as<long long>(),
                                                            W->inv_v2.as<unsigned long long>(), W->qoff.as<long long>(),
                                                            q0, q1, qo[q0], n_gal, W->pk.as<unsigned long long>(),
                                                            W->pv.as<float>());
      IBL_CUDA_OK(cudaGetLastError());
      int key_bits = 1;
      while ((1ull << key_bits) < (unsigned long long)(q1 - q0) * (unsigned long long)n_gal) ++key_bits;
      size_t tb = 0;
      IBL_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, tb, W->pk.as<unsigned long long>(),
                                                  W->pk2.as<unsigned long long>(), W->pv.as<float>(), W->pv2.as<float>(),
                                                  T, 0, key_bits, s));
      IBL_RET(W->temp.ensure(tb + 256));
      IBL_CUDA_OK(cub::DeviceRadixSort::SortPairs(W->temp.p, tb, W->pk.as<unsigned long long>(),
                                                  W->pk2.as<unsigned long long>(), W->pv.as<float>(), W->pv2.as<float>(),
                                                  T, 0, key_bits, s));
      rr_segment_sum_kernel<<<cdiv(T, 256), 256, 0, s>>>(W->pk2.as<unsigned long long>(), W->pv2.as<float>(), T,
                                                         W->tsum.as<float>());
      IBL_CUDA_OK(cudaGetLastError());
      nl += 3;
    }
    IBL_RET(emit(q0, q1, qo[q0], T));
    q0 = q1;
  }
  return IBL_OK;
}

int launch_rerank_topk(RerankWs* W, const float* X, int N, int m, int d, const long long* nbr, const float* nbr_dist,
                       int w, const float* rowmax, int k1, int k2, float lam, const long long* orig, int k_orig, int k,
                       float* out_dist, long long* out_idx, uint64_t* launches, cudaStream_t s) {
  const long long n_gal = (long long)N - m;
  uint64_t nl = 0;
  // the exact routine wants rows of a multiple of 4 floats
  const int dp = (d + 3) / 4 * 4;
  const float* x = X;
  if (dp != d) {
    IBL_RET(W->xpad.ensure((size_t)N * dp * 4));
    IBL_CUDA_OK(cudaMemsetAsync(W->xpad.p, 0, (size_t)N * dp * 4, s));
    IBL_CUDA_OK(cudaMemcpy2DAsync(W->xpad.p, (size_t)dp * 4, X, (size_t)d * 4, (size_t)d * 4, N, cudaMemcpyDeviceToDevice, s));
    x = W->xpad.as<float>();
  }
  IBL_RET(W->sq.ensure((size_t)N * 4));
  rr_sqnorm_kernel<<<N, 256, 0, s>>>(x, dp, W->sq.as<float>());
  ExpandArgs ea{};
  ea.x = x; ea.d = dp; ea.sq = W->sq.as<float>(); ea.nbr = nbr; ea.nbr_dist = nbr_dist; ea.w = w; ea.rowmax = rowmax;
  const float oml = (float)(1.0 - (double)lam);  // numpy casts the scalar (1 - lambda) to float32
  IBL_RET(rerank_sparse<false>(W, ea, N, m, k1, k2, nl, s, [&](int q0, int q1, long long base, long long) -> int {
    TopkArgs ta{};
    ta.x = x; ta.d = dp; ta.sq = W->sq.as<float>(); ta.rowmax = rowmax; ta.m = m; ta.n_gal = n_gal;
    ta.keys = W->pk2.as<unsigned long long>(); ta.t = W->tsum.as<float>(); ta.qoff = W->qoff.as<long long>();
    ta.base = base; ta.q0 = q0; ta.orig = orig; ta.k_orig = k_orig; ta.lam = lam; ta.oml = oml; ta.k = k;
    ta.out_dist = out_dist; ta.out_idx = out_idx;
    rr_topk_kernel<<<q1 - q0, 256, 0, s>>>(ta);
    IBL_CUDA_OK(cudaGetLastError());
    nl += 1;
    return IBL_OK;
  }));
  if (launches) *launches += nl;
  return IBL_OK;
}

int launch_rerank_dense(RerankWs* W, const float* qg, const float* qq, const float* gg, int m, int n, int k1, int k2,
                        double lam, float* out, uint64_t* launches, cudaStream_t s) {
  const int N = m + n, w = std::max(k1 + 1, k2);
  IBL_REQUIRE(w <= 128 && w <= N, "dense re-ranking: max(k1 + 1, k2) <= min(128, m + n)");
  IBL_RET(rr_set_attributes<true>());
  uint64_t nl = 0;
  // neighbour lists [N,w] int64, their D[j][i] [N,w] and M [N]
  IBL_RET(W->dn.ensure((size_t)N * w * 12 + (size_t)N * 4));
  long long* nbr = W->dn.as<long long>();
  float* nd = reinterpret_cast<float*>(nbr + (size_t)N * w);
  float* mx = nd + (size_t)N * w;
  const DenseSrc src{qg, qq, gg, m, n};
  dn_knn_kernel<<<cdiv(N, 32), DN_WARPS * 32, dn_knn_smem(w), s>>>(src, w, nbr, nd, mx);
  IBL_CUDA_OK(cudaGetLastError());
  // 1 - lambda in double, then float32: numpy's (1 - lambda_value) is a Python float cast to the array's type
  const float c1 = (float)(1.0 - lam), c2 = (float)lam;
  rr_dense_base_kernel<<<std::min(cdiv((long long)m * n, 256), 32 * device_sm_count()), 256, 0, s>>>(qg, mx, m, n, c1,
                                                                                                      c2, out);
  IBL_CUDA_OK(cudaGetLastError());
  nl += 2;
  ExpandArgs ea{};
  ea.sq = mx;   // not read with a dense source; a valid pointer all the same
  ea.nbr = nbr; ea.nbr_dist = nd; ea.w = w; ea.rowmax = mx; ea.dn = src;
  IBL_RET(rerank_sparse<true>(W, ea, N, m, k1, k2, nl, s, [&](int q0, int, long long, long long T) -> int {
    if (T == 0) return IBL_OK;
    rr_dense_scatter_kernel<<<cdiv(T, 256), 256, 0, s>>>(W->pk2.as<unsigned long long>(), W->tsum.as<float>(), T, q0,
                                                         n, qg, mx, c1, c2, out);
    IBL_CUDA_OK(cudaGetLastError());
    nl += 1;
    return IBL_OK;
  }));
  if (launches) *launches += nl;
  return IBL_OK;
}

}  // namespace ibl
