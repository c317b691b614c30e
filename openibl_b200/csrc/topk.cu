// Per-query top-k selection and k-way merge (replaces np.argsort over the full distance row,
// reference ibl/evaluators.py:143; only the first 10 (120 with nms) ranks are read, :151-159).
// Order is (distance, index) ascending: ties go to the lowest database index.
#include "common.cuh"
#include "ranking.cuh"

namespace ibl {

constexpr int TK_PER_ITER = 1024; // elements examined per block iteration (4 per thread)
constexpr unsigned long long TK_MAX = ~0ull;

// One block per query row.  buf[0,k) holds the best k keys found so far (after a compaction), buf[k, k+cnt)
// the candidates appended since.  CAP = 2048 serves k <= 128, CAP = 4096 serves k <= 1024 (the reference's
// evaluate_all accepts any recall_topk, evaluators.py:142-153).  Invariant before every iteration:
// k + cnt + TK_PER_ITER <= CAP.
// blockIdx.y selects a segment of `seg` columns: a row split over several blocks writes one sorted list per segment,
// out_* [segments][m][k], with the segment's first column added to idx_base (one segment: the whole row).
template <int CAP>
__global__ void __launch_bounds__(256)
topk_rows_kernel(const float* __restrict__ dist, long long ld, int n_valid, int k,
                 long long idx_base, float* __restrict__ out_dist,
                 long long* __restrict__ out_idx, int seg = 0) {
  __shared__ unsigned long long buf[CAP];
  __shared__ int cnt;
  __shared__ unsigned long long thr_s;
  const long long row = blockIdx.x;
  const float* d = dist + row * ld;
  if (gridDim.y > 1) {
    const int c0 = blockIdx.y * seg;
    d += c0;
    idx_base += c0;
    n_valid = min(seg, n_valid - c0);
    out_dist += (long long)blockIdx.y * gridDim.x * k;
    out_idx += (long long)blockIdx.y * gridDim.x * k;
  }
  for (int i = threadIdx.x; i < CAP; i += blockDim.x) buf[i] = TK_MAX;
  if (threadIdx.x == 0) { cnt = 0; thr_s = TK_MAX; }
  __syncthreads();

  for (int j0 = 0; j0 < n_valid; j0 += TK_PER_ITER) {
    const unsigned long long thr = thr_s;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u * 256 + threadIdx.x;
      if (j < n_valid) {
        const unsigned long long key = rank_key(__ldg(d + j), (unsigned)j);
        if (key < thr) {
          const int pos = atomicAdd(&cnt, 1);
          buf[k + pos] = key;
        }
      }
    }
    __syncthreads();
    // Every thread takes the SAME snapshot of cnt, and nobody starts the next iteration's atomicAdd before
    // all have read it: the branch below contains barriers, so it must be block-uniform.
    const int c = cnt;
    __syncthreads();
    if (k + c + TK_PER_ITER > CAP) {
      block_bitonic_sort(buf, CAP);
      for (int i = k + threadIdx.x; i < CAP; i += blockDim.x) buf[i] = TK_MAX;
      if (threadIdx.x == 0) { cnt = 0; thr_s = buf[k - 1]; }
      __syncthreads();
    }
  }
  block_bitonic_sort(buf, CAP);
  for (int i = threadIdx.x; i < k; i += blockDim.x) store_ranked(buf[i], idx_base, out_dist, out_idx, row * k + i);
}

int launch_topk_rows(const float* dist, long long ld, int m, int n_valid, int k, int64_t idx_base,
                     float* out_dist, int64_t* out_idx, bool accumulate, cudaStream_t s) {
  (void)accumulate;
  IBL_REQUIRE(k >= 1 && k <= 1024, "top-k supports 1 <= k <= 1024");
  if (m == 0) return IBL_OK;
  if (k <= 128)
    topk_rows_kernel<2048><<<m, 256, 0, s>>>(dist, ld, n_valid, k, (long long)idx_base, out_dist,
                                             reinterpret_cast<long long*>(out_idx));
  else
    topk_rows_kernel<4096><<<m, 256, 0, s>>>(dist, ld, n_valid, k, (long long)idx_base, out_dist,
                                             reinterpret_cast<long long*>(out_idx));
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// Per-row top-k of dist [m][n_valid] (row stride ld) in `segs` segments of `seg` columns (segs * seg >= n_valid):
// out_* [segs][m][k], each list ascending by (distance, index), indices idx_base + column
int launch_topk_rows_seg(const float* dist, long long ld, int m, int n_valid, int k, int segs, int seg,
                         int64_t idx_base, float* out_dist, int64_t* out_idx, cudaStream_t s) {
  IBL_REQUIRE(k >= 1 && k <= 128 && segs >= 1 && (long long)segs * seg >= n_valid &&
                  (long long)(segs - 1) * seg < n_valid,
              "segmented top-k: 1 <= k <= 128, the segments cover the row");
  if (m == 0) return IBL_OK;
  topk_rows_kernel<2048><<<dim3(m, segs), 256, 0, s>>>(dist, ld, n_valid, k, (long long)idx_base, out_dist,
                                                      reinterpret_cast<long long*>(out_idx), seg);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

// ---- merge of per-shard candidate lists -------------------------------------------------------
// one block per query; candidates sorted by (dist, idx) with a two-array bitonic network
__global__ void __launch_bounds__(256)
topk_merge_kernel(const float* __restrict__ cand_dist, const long long* __restrict__ cand_idx,
                  int parts, int m, int k_in, int k_out, int cap /*pow2 >= parts*k_in*/,
                  float* __restrict__ out_dist, long long* __restrict__ out_idx) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  long long* sidx = reinterpret_cast<long long*>(smem_raw);
  uint32_t* skey = reinterpret_cast<uint32_t*>(sidx + cap);
  const long long row = blockIdx.x;
  const int total = parts * k_in;
  for (int i = threadIdx.x; i < cap; i += blockDim.x) {
    uint32_t key = 0xffffffffu;
    long long idx = 0x7fffffffffffffffll;
    if (i < total) {
      const int p = i / k_in, j = i - p * k_in;
      const long long src = ((long long)p * m + row) * k_in + j;
      const long long ci = cand_idx[src];
      if (ci >= 0) { key = ord_key(cand_dist[src]); idx = ci; }
    }
    skey[i] = key;
    sidx[i] = idx;
  }
  for (int size = 2; size <= cap; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < (cap >> 1); i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const uint32_t ka = skey[lo], kb = skey[hi];
        const long long ia = sidx[lo], ib = sidx[hi];
        const bool gt = (ka > kb) || (ka == kb && ia > ib);
        if (gt == up) { skey[lo] = kb; skey[hi] = ka; sidx[lo] = ib; sidx[hi] = ia; }
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < k_out; i += blockDim.x) {
    const bool valid = (i < cap) && sidx[i] != 0x7fffffffffffffffll;
    out_dist[row * k_out + i] = valid ? unord_key(skey[i]) : INFINITY;
    out_idx[row * k_out + i] = valid ? sidx[i] : -1;
  }
}

int launch_topk_merge(const float* cand_dist, const int64_t* cand_idx, int parts, int m, int k_in,
                      int k_out, float* out_dist, int64_t* out_idx, cudaStream_t s) {
  const int total = parts * k_in;
  IBL_REQUIRE(total >= 1 && total <= 8192, "topk_merge supports up to 8192 candidates per query");
  IBL_REQUIRE(k_out >= 1 && k_out <= total, "topk_merge: 1 <= k_out <= parts*k_in");
  int cap = 2;
  while (cap < total) cap <<= 1;
  const size_t smem = (size_t)cap * (sizeof(long long) + sizeof(uint32_t));
  static DeviceOnce attr_set;   // the attribute is per device
  if (!attr_set.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(topk_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     8192 * 12));
    attr_set.mark();
  }
  if (m == 0) return IBL_OK;
  topk_merge_kernel<<<m, 256, smem, s>>>(cand_dist, reinterpret_cast<const long long*>(cand_idx),
                                         parts, m, k_in, k_out, cap, out_dist,
                                         reinterpret_cast<long long*>(out_idx));
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

}  // namespace ibl
