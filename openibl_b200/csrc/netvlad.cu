// NetVLAD aggregation (reference ibl/models/netvlad.py:44-61) and the EmbedNet normalisations
// (netvlad.py:78-80) on CUDA cores, fp32.
//
//   x^[s,:]   = x[s,:] / max(|x[s,:]|, 1e-12)                       (netvlad.py:47)
//   a[s,:]    = softmax_k( W x^[s,:] )                              (netvlad.py:50-51)
//   vlad[k,c] = sum_s a[s,k] x^[s,c]  -  cent[k,c] * sum_s a[s,k]   (netvlad.py:56-59, expanded)
//
// The reference materialises a [N,K,C,S] residual tensor (157 MB / image); here the two
// contractions are tiled GEMMs and nothing larger than [N,S,K] is written.
//
// The blocks are 64 clusters wide.  K < 64 clusters run on the same blocks: clusters K..63 get zero weights and are
// left out of the softmax, so their assignment is 0; assign and the outputs are stored at a stride of K.
#include "common.cuh"

namespace ibl {

constexpr int NV_K = 64;  // clusters handled per block: the most the kernels serve (the reference default)

// element (n,s,c) of the feature map for both supported layouts
struct FeatView {
  const float* p;
  long long sN, sS, sC;
  __device__ __forceinline__ float at(long long n, int s, int c) const {
    return __ldg(p + n * sN + s * sS + c * sC);
  }
};

// ---- kernel A: per-pixel inverse norm + soft-assignment -----------------------------------
// block = 32 pixels x 64 clusters, 256 threads: thread (p = t%32, kg = t/32) owns 8 logits.
__global__ void __launch_bounds__(256)
netvlad_assign_kernel(FeatView f, bool nhwc, int C, int S, const float* __restrict__ w /*[K][C]*/, int K,
                      int normalize_input, float* __restrict__ assign /*[N,S,K]*/,
                      float* __restrict__ invnorm /*[N,S]*/) {
  __shared__ float xs[32][65];
  __shared__ float wsm[NV_K][65];
  __shared__ float zs[32][65];
  __shared__ float inv_s[32];
  const int t = threadIdx.x;
  const int p = t & 31, kg = t >> 5;
  const long long n = blockIdx.y;
  const int s0 = blockIdx.x * 32;

  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  float ss = 0.f;

  for (int c0 = 0; c0 < C; c0 += 64) {
    for (int e = t; e < 32 * 64; e += 256) {
      int pp, cc;
      if (nhwc) { pp = e >> 6; cc = e & 63; } else { cc = e >> 5; pp = e & 31; }
      const int s = s0 + pp, c = c0 + cc;
      xs[pp][cc] = (s < S && c < C) ? f.at(n, s, c) : 0.f;
    }
    for (int e = t; e < NV_K * 64; e += 256) {
      const int k = e >> 6, cc = e & 63;
      wsm[k][cc] = (k < K && c0 + cc < C) ? __ldg(w + (long long)k * C + c0 + cc) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int cc = 0; cc < 64; ++cc) {
      const float xv = xs[p][cc];
      ss = fmaf(xv, xv, ss);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(xv, wsm[kg * 8 + j][cc], acc[j]);
    }
    __syncthreads();
  }
  float inv = 1.f;
  if (normalize_input) inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  if (kg == 0) inv_s[p] = inv;
#pragma unroll
  for (int j = 0; j < 8; ++j) zs[p][kg * 8 + j] = acc[j] * inv;
  __syncthreads();

  // softmax over the K clusters: warp w handles pixels 4w..4w+3, two clusters per lane
  const int lane = t & 31, wid = t >> 5;
  for (int q = 0; q < 4; ++q) {
    const int pp = wid * 4 + q;
    const int s = s0 + pp;
    float z0 = zs[pp][lane], z1 = zs[pp][lane + 32];
    if (lane >= K) z0 = -INFINITY;
    if (lane + 32 >= K) z1 = -INFINITY;
    float m = fmaxf(z0, z1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const float e0 = expf(z0 - m), e1 = expf(z1 - m);
    float sum = e0 + e1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (s < S) {
      float* ap = assign + (n * S + s) * (long long)K;
      if (lane < K) ap[lane] = e0 / sum;
      if (lane + 32 < K) ap[lane + 32] = e1 / sum;
      if (lane == 0) invnorm[n * S + s] = inv_s[pp];
    }
  }
}

// ---- kernel B: vlad[k,c] = sum_s a[s,k] (x[s,c] inv[s]) - cent[k,c] asum[k] -----------------
// block = 64 clusters x 64 channels, 256 threads, 4x4 per thread, S in chunks of 16.
__global__ void __launch_bounds__(256)
netvlad_aggregate_kernel(FeatView f, bool nhwc, int C, int S, int K, const float* __restrict__ assign,
                         const float* __restrict__ invnorm, const float* __restrict__ cent,
                         float* __restrict__ raw /*[N,K,C]*/) {
  __shared__ __align__(16) float As[16][NV_K];
  __shared__ __align__(16) float Bs[16][64];
  const int t = threadIdx.x;
  const int tn = t & 15, tm = t >> 4;
  const long long n = blockIdx.y;
  const int c0 = blockIdx.x * 64;
  float acc[4][4];
  float asum[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    asum[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  }
  for (int sb = 0; sb < S; sb += 16) {
    for (int e = t; e < 16 * 64; e += 256) {
      const int ss = e >> 6, k = e & 63;
      const int s = sb + ss;
      As[ss][k] = (s < S && k < K) ? __ldg(assign + (n * S + s) * (long long)K + k) : 0.f;
    }
    for (int e = t; e < 16 * 64; e += 256) {
      int ss, cc;
      if (nhwc) { ss = e >> 6; cc = e & 63; } else { cc = e >> 4; ss = e & 15; }
      const int s = sb + ss, c = c0 + cc;
      float v = 0.f;
      if (s < S && c < C) v = f.at(n, s, c) * __ldg(invnorm + n * S + s);
      Bs[ss][cc] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][tm * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tn * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        asum[i] += av[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = tm * 4 + i;
    if (k >= K) break;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + tn * 4 + j;
      if (c < C) raw[(n * K + k) * (long long)C + c] = acc[i][j] - __ldg(cent + (long long)k * C + c) * asum[i];
    }
  }
}

// ---- kernel C: intra-normalise rows, flatten, global L2 (netvlad.py:78-80) ------------------
__global__ void __launch_bounds__(256)
vlad_normalize_kernel(const float* __restrict__ raw, int K, int C, float* __restrict__ out) {
  extern __shared__ float sm[];  // row_inv[K], row_ss[K]
  float* row_inv = sm;
  float* row_ss = sm + K;
  __shared__ float ginv_s;
  const long long n = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* r = raw + n * (long long)K * C;
  for (int k = wid; k < K; k += nw) {
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = r[(long long)k * C + c]; ss = fmaf(v, v, ss); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
    float s2 = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = r[(long long)k * C + c] * inv; s2 = fmaf(v, v, s2); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    if (lane == 0) { row_inv[k] = inv; row_ss[k] = s2; }
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    float tot = 0.f;
    for (int k = lane; k < K; k += 32) tot += row_ss[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
    if (lane == 0) ginv_s = 1.f / fmaxf(sqrtf(tot), 1e-12f);
  }
  __syncthreads();
  const float ginv = ginv_s;
  float* o = out + n * (long long)K * C;
  const int total = K * C;
  for (int e = threadIdx.x; e < total; e += blockDim.x) o[e] = r[e] * row_inv[e / C] * ginv;
}

int launch_vlad_normalize(const float* raw, int N, int K, int C, float* out, cudaStream_t s) {
  vlad_normalize_kernel<<<N, 256, 2 * K * sizeof(float), s>>>(raw, K, C, out);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}

int launch_netvlad(const float* feat, bool nhwc, int N, int C, int S, const float* conv_w,
                   const float* centroids, int K, bool normalize_input, float* assign,
                   float* invnorm, float* asum, float* vlad_raw, float* vlad_norm,
                   cudaStream_t s, uint64_t* launches) {
  (void)asum;
  IBL_REQUIRE(K >= 1 && K <= NV_K, "NetVLAD kernels serve 1..64 clusters");
  FeatView f;
  f.p = feat;
  f.sN = (long long)S * C;
  if (nhwc) { f.sS = C; f.sC = 1; } else { f.sS = 1; f.sC = S; }
  dim3 ga((unsigned)cdiv(S, 32), (unsigned)N);
  netvlad_assign_kernel<<<ga, 256, 0, s>>>(f, nhwc, C, S, conv_w, K, normalize_input ? 1 : 0, assign, invnorm);
  IBL_CUDA_OK(cudaGetLastError());
  dim3 gb((unsigned)cdiv(C, 64), (unsigned)N);
  netvlad_aggregate_kernel<<<gb, 256, 0, s>>>(f, nhwc, C, S, K, assign, invnorm, centroids, vlad_raw);
  IBL_CUDA_OK(cudaGetLastError());
  *launches += 2;
  if (vlad_norm) {
    IBL_RET(launch_vlad_normalize(vlad_raw, N, K, C, vlad_norm, s));
    *launches += 1;
  }
  return IBL_OK;
}

}  // namespace ibl

namespace ibl {
// soft-assignment + inverse norms only (shared with the backward pass, netvlad_bwd.cu)
int launch_netvlad_assign(const float* feat, bool nhwc, int N, int C, int S, const float* conv_w, int K,
                          bool normalize_input, float* assign, float* invnorm, cudaStream_t s) {
  IBL_REQUIRE(K >= 1 && K <= NV_K, "NetVLAD kernels serve 1..64 clusters");
  FeatView f;
  f.p = feat;
  f.sN = (long long)S * C;
  if (nhwc) { f.sS = C; f.sC = 1; } else { f.sS = 1; f.sC = S; }
  dim3 ga((unsigned)cdiv(S, 32), (unsigned)N);
  netvlad_assign_kernel<<<ga, 256, 0, s>>>(f, nhwc, C, S, conv_w, K, normalize_input ? 1 : 0, assign, invnorm);
  IBL_CUDA_OK(cudaGetLastError());
  return IBL_OK;
}
}  // namespace ibl
