// Full ascending argsort of every row of a distance matrix on the device (SURVEY 8 f3: the training samplers'
// hard-negative mining starts with `torch.argsort(distmat, dim=1)` on the CPU, reference
// ibl/utils/data/sampler.py:46-54,126-135).  Order: (distance, index) ascending -- the stable order.
//
//   n <= 16384        one block per row: keys (orderable fp32 << 32 | column) in shared memory, bitonic network
//   n  > 16384        the same per 16384-column chunk, then log2(chunks) merge passes in global memory; each element
//                     finds its merged position with one binary search in the sibling run (keys are unique, so
//                     lower_bound on one side and on the other give a stable, collision-free scatter)
#include "common.cuh"
#include "ranking.cuh"

namespace ibl {

constexpr int SR_CHUNK = 16384;

// grid (chunks, m); sorts columns [c*SR_CHUNK, ...) of row r; writes u64 keys (runs) or final int64 indices
__global__ void __launch_bounds__(1024)
sort_chunk_kernel(const float* __restrict__ dist, long long ld, int n, unsigned long long* __restrict__ keys_out,
                  long long* __restrict__ idx_out, int cap /*pow2 >= chunk length, <= SR_CHUNK*/) {
  extern __shared__ unsigned long long sk[];
  const long long r = blockIdx.y;
  const int c0 = blockIdx.x * SR_CHUNK;
  const int len = min(SR_CHUNK, n - c0);
  const float* d = dist + r * ld + c0;
  for (int i = threadIdx.x; i < cap; i += blockDim.x)
    sk[i] = i < len ? rank_key(d[i], (unsigned)(c0 + i)) : ~0ull;
  block_bitonic_sort(sk, cap);
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
    if (idx_out) idx_out[r * n + c0 + i] = (long long)(uint32_t)(sk[i] & 0xffffffffu);
    else keys_out[r * n + c0 + i] = sk[i];
  }
}

// one merge pass: runs of length `run` -> runs of length 2*run.  grid (ceil(n/256), m)
__global__ void __launch_bounds__(256)
merge_pass_kernel(const unsigned long long* __restrict__ src, int n, int run, unsigned long long* __restrict__ dst,
                  long long* __restrict__ idx_out /*last pass only*/) {
  const long long r = blockIdx.y;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const unsigned long long* row = src + r * n;
  const int pair0 = (i / (2 * run)) * (2 * run);
  const int a0 = pair0, a1 = min(n, pair0 + run), b0 = a1, b1 = min(n, pair0 + 2 * run);
  const unsigned long long key = row[i];
  int lo, hi, base;
  if (i < a1) { lo = b0; hi = b1; base = i - a0; }          // element of run A: count B elements < key
  else { lo = a0; hi = a1; base = i - b0; }                 // element of run B: count A elements < key (unique keys)
  const int s0 = lo;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (row[mid] < key) lo = mid + 1; else hi = mid;
  }
  const int pos = pair0 + base + (lo - s0);
  if (idx_out) idx_out[r * n + pos] = (long long)(uint32_t)(key & 0xffffffffu);
  else dst[r * n + pos] = key;
}

// dist [m, n] (row stride ld) -> idx [m, n] int64.  scratch: 2 * m * n u64 when n > SR_CHUNK, unused otherwise.
int launch_argsort_rows(const float* dist, long long ld, int m, int n, long long* idx, unsigned long long* scratch,
                        cudaStream_t s, uint64_t* launches) {
  if (m == 0 || n == 0) return IBL_OK;
  static DeviceOnce attr_done;
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(sort_chunk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SR_CHUNK * 8));
    attr_done.mark();
  }
  const int chunks = cdiv(n, SR_CHUNK);
  int cap = 2;
  while (cap < (n < SR_CHUNK ? n : SR_CHUNK)) cap <<= 1;
  if (chunks == 1) {
    sort_chunk_kernel<<<dim3(1, m), 1024, (size_t)cap * 8, s>>>(dist, ld, n, nullptr, idx, cap);
    IBL_CUDA_OK(cudaGetLastError());
    if (launches) ++*launches;
    return IBL_OK;
  }
  IBL_REQUIRE(scratch, "argsort of rows longer than 16384 needs the merge scratch");
  unsigned long long* a = scratch;
  unsigned long long* b = scratch + (size_t)m * n;
  sort_chunk_kernel<<<dim3(chunks, m), 1024, (size_t)SR_CHUNK * 8, s>>>(dist, ld, n, a, nullptr, SR_CHUNK);
  if (launches) ++*launches;
  for (int run = SR_CHUNK; run < n; run <<= 1) {
    const bool lastp = 2ll * run >= n;
    merge_pass_kernel<<<dim3(cdiv(n, 256), m), 256, 0, s>>>(a, n, run, b, lastp ? idx : nullptr);
    if (launches) ++*launches;
    unsigned long long* t = a; a = b; b = t;
  }
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

}  // namespace ibl
