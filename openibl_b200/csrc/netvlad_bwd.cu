// NetVLAD backward (SURVEY 8 row a11: what autograd computes for ibl/models/netvlad.py:44-61 when the SFRS
// trainer back-propagates through EmbedRegionNet, netvlad.py:139-146 / trainers.py:235-259).  fp32 CUDA cores.
//
// forward   x^ = x / max(|x|, eps),  z = W x^,  a = softmax_k z,  vlad[k,c] = sum_s a[s,k] (x^[s,c] - cent[k,c])
// given     g[k,c] = dL/dvlad[k,c]
//   dcent[k,c] = - sum_n g[n,k,c] * sum_s a[n,s,k]
//   da[s,k]    = x^[s,:].g[k,:] - g[k,:].cent[k,:]
//   dz[s,k]    = a[s,k] (da[s,k] - sum_j a[s,j] da[s,j])
//   dW[k,c]    = sum_{n,s} dz[n,s,k] x^[n,s,c]
//   dx^[s,c]   = sum_k a[s,k] g[k,c] + dz[s,k] W[k,c]
//   dx[s,c]    = (dx^[s,c] - x^[s,c] (x^[s,:].dx^[s,:])) / max(|x[s,:]|, eps)        (normalize_input)
//
// The soft-assignment a and 1/|x| are recomputed with the forward's assign kernel instead of being
// saved (the reference's autograd keeps the [N,K,C,S] residual tensor alive for backward).
//
// The blocks are 64 clusters wide; for K < 64 clusters K..63 load zeros (a, dz, g, W, cent), so they add nothing, and
// every [.., K] / [K, C] tensor is read and written at a stride of K.
#include "common.cuh"

namespace ibl {

constexpr int NB_K = 64;   // clusters per block: the most the kernels serve

struct FeatV {
  const float* p;
  long long sN, sS, sC;
  __device__ __forceinline__ float at(long long n, int s, int c) const { return __ldg(p + n * sN + s * sS + c * sC); }
};

// ---- dz[n,s,k] and asum[n,k] --------------------------------------------------------------------
// block = 32 pixels x 64 clusters (256 threads: thread (p = t%32, kg = t/32) owns 8 clusters)
__global__ void __launch_bounds__(256)
nv_bwd_dz_kernel(FeatV f, bool nhwc, int C, int S, int K, const float* __restrict__ g /*[N,K,C]*/,
                 const float* __restrict__ cent, const float* __restrict__ assign /*[N,S,K]*/,
                 const float* __restrict__ invnorm /*[N,S]*/, float* __restrict__ dz /*[N,S,K]*/) {
  __shared__ float xs[32][65];
  __shared__ float gs[NB_K][65];
  __shared__ float ps[32][65];
  __shared__ float gc[NB_K];
  const int t = threadIdx.x, p = t & 31, kg = t >> 5;
  const long long n = blockIdx.y;
  const int s0 = blockIdx.x * 32;
  const float* gn = g + n * K * (long long)C;
  // gc[k] = g[k,:].cent[k,:]  (4 threads per cluster)
  {
    const int k = t >> 2, part = t & 3;
    float acc = 0.f;
    if (k < K)
      for (int c = part; c < C; c += 4) acc = fmaf(__ldg(gn + (long long)k * C + c), __ldg(cent + (long long)k * C + c), acc);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    if (part == 0) gc[k] = acc;
  }
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int c0 = 0; c0 < C; c0 += 64) {
    __syncthreads();
    for (int e = t; e < 32 * 64; e += 256) {
      int pp, cc;
      if (nhwc) { pp = e >> 6; cc = e & 63; } else { cc = e >> 5; pp = e & 31; }
      const int s = s0 + pp, c = c0 + cc;
      xs[pp][cc] = (s < S && c < C) ? f.at(n, s, c) * __ldg(invnorm + n * S + s) : 0.f;
    }
    for (int e = t; e < NB_K * 64; e += 256) {
      const int k = e >> 6, cc = e & 63;
      gs[k][cc] = (k < K && c0 + cc < C) ? __ldg(gn + (long long)k * C + c0 + cc) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int cc = 0; cc < 64; ++cc) {
      const float xv = xs[p][cc];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(xv, gs[kg * 8 + j][cc], acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) ps[p][kg * 8 + j] = acc[j] - gc[kg * 8 + j];   // da[s,k]
  __syncthreads();
  // softmax backward: warp w handles pixels 4w..4w+3, two clusters per lane
  const int lane = t & 31, wid = t >> 5;
  for (int q = 0; q < 4; ++q) {
    const int pp = wid * 4 + q, s = s0 + pp;
    if (s >= S) continue;                         // warp-uniform
    const float* ap = assign + (n * S + s) * (long long)K;
    const float a0 = lane < K ? __ldg(ap + lane) : 0.f, a1 = lane + 32 < K ? __ldg(ap + lane + 32) : 0.f;
    const float d0 = ps[pp][lane], d1 = ps[pp][lane + 32];
    float tsum = a0 * d0 + a1 * d1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tsum += __shfl_xor_sync(0xffffffffu, tsum, o);
    float* o = dz + (n * S + s) * (long long)K;
    if (lane < K) o[lane] = a0 * (d0 - tsum);
    if (lane + 32 < K) o[lane + 32] = a1 * (d1 - tsum);
  }
}

// ---- dx: one block per 32 pixels, all channels kept in shared memory ---------------------------------
// dx^[s,c] = sum_k a[s,k] g[k,c] + dz[s,k] W[k,c];  dx = inv (dx^ - x^ (x^.dx^))
__global__ void __launch_bounds__(256)
nv_bwd_dx_kernel(FeatV f, bool nhwc, int C, int S, int K, const float* __restrict__ g, const float* __restrict__ w,
                 const float* __restrict__ assign, const float* __restrict__ dz,
                 const float* __restrict__ invnorm, int normalize_input, float* __restrict__ dx,
                 long long dN, long long dS, long long dC) {
  extern __shared__ float sm[];
  float* a_t = sm;                     // [32][65]
  float* z_t = a_t + 32 * 65;          // [32][65]
  float* g_t = z_t + 32 * 65;          // [64][65]   g[k][c chunk]
  float* w_t = g_t + 64 * 65;          // [64][65]
  float* dxh = w_t + 64 * 65;          // [32][C+1]
  __shared__ float rdot[32];
  const int t = threadIdx.x, p = t & 31, cg = t >> 5;   // thread owns pixel p, channels cg*8..+8 of the chunk
  const long long n = blockIdx.y;
  const int s0 = blockIdx.x * 32;
  const int ldx = C + 1;
  for (int e = t; e < 32 * 64; e += 256) {
    const int pp = e >> 6, k = e & 63, s = s0 + pp;
    a_t[pp * 65 + k] = (s < S && k < K) ? __ldg(assign + (n * S + s) * (long long)K + k) : 0.f;
    z_t[pp * 65 + k] = (s < S && k < K) ? __ldg(dz + (n * S + s) * (long long)K + k) : 0.f;
  }
  const float* gn = g + n * K * (long long)C;
  for (int c0 = 0; c0 < C; c0 += 64) {
    __syncthreads();
    for (int e = t; e < NB_K * 64; e += 256) {
      const int k = e >> 6, cc = e & 63;
      const bool ok = k < K && c0 + cc < C;
      g_t[k * 65 + cc] = ok ? __ldg(gn + (long long)k * C + c0 + cc) : 0.f;
      w_t[k * 65 + cc] = ok ? __ldg(w + (long long)k * C + c0 + cc) : 0.f;
    }
    __syncthreads();
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll 4
    for (int k = 0; k < NB_K; ++k) {
      const float av = a_t[p * 65 + k], zv = z_t[p * 65 + k];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        acc[j] = fmaf(av, g_t[k * 65 + cg * 8 + j], fmaf(zv, w_t[k * 65 + cg * 8 + j], acc[j]));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) dxh[p * ldx + c0 + cg * 8 + j] = acc[j];
  }
  __syncthreads();
  // r[s] = x^[s,:].dx^[s,:]   (warp w handles pixels 4w..4w+3)
  const int lane = t & 31, wid = t >> 5;
  for (int q = 0; q < 4; ++q) {
    const int pp = wid * 4 + q, s = s0 + pp;
    float r = 0.f;
    if (s < S && normalize_input) {
      const float inv = __ldg(invnorm + n * S + s);
      for (int c = lane; c < C; c += 32) r = fmaf(f.at(n, s, c) * inv, dxh[pp * ldx + c], r);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    if (lane == 0) rdot[pp] = r;
  }
  __syncthreads();
  for (int e = t; e < 32 * C; e += 256) {
    int pp, c;
    if (nhwc) { pp = e / C; c = e - pp * C; } else { c = e >> 5; pp = e & 31; }
    const int s = s0 + pp;
    if (s >= S) continue;
    float v = dxh[pp * ldx + c];
    if (normalize_input) {
      const float inv = __ldg(invnorm + n * S + s);
      v = inv * (v - f.at(n, s, c) * inv * rdot[pp]);
    }
    dx[n * dN + s * dS + c * dC] = v;
  }
}

// ---- dW partials: part[z][k][c] = sum over the z-th slice of (n,s) of dz[n,s,k] x^[n,s,c] ------------
// block = 64 clusters x 64 channels, 4x4 per thread; grid (C/64, splits)
__global__ void __launch_bounds__(256)
nv_bwd_dw_kernel(FeatV f, bool nhwc, int C, int S, int N, int K, const float* __restrict__ dz,
                 const float* __restrict__ invnorm, int rows_per_split, float* __restrict__ part) {
  __shared__ __align__(16) float As[16][NB_K];
  __shared__ __align__(16) float Bs[16][64];
  const int t = threadIdx.x, tn = t & 15, tm = t >> 4;
  const int c0 = blockIdx.x * 64;
  const long long R = (long long)N * S;
  const long long r0 = (long long)blockIdx.y * rows_per_split;
  const long long r1 = (r0 + rows_per_split < R) ? r0 + rows_per_split : R;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (long long rb = r0; rb < r1; rb += 16) {
    for (int e = t; e < 16 * 64; e += 256) {
      const int rr = e >> 6, k = e & 63;
      const long long r = rb + rr;
      As[rr][k] = (r < r1 && k < K) ? __ldg(dz + r * K + k) : 0.f;
    }
    for (int e = t; e < 16 * 64; e += 256) {
      int rr, cc;
      if (nhwc) { rr = e >> 6; cc = e & 63; } else { cc = e >> 4; rr = e & 15; }
      const long long r = rb + rr;
      float v = 0.f;
      if (r < r1 && c0 + cc < C) {
        const long long n = r / S;
        const int s = (int)(r - n * S);
        v = f.at(n, s, c0 + cc) * __ldg(invnorm + r);
      }
      Bs[rr][cc] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][tm * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tn * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* o = part + (long long)blockIdx.y * K * C;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + tn * 4 + j;
      if (tm * 4 + i < K && c < C) o[(long long)(tm * 4 + i) * C + c] = acc[i][j];
    }
}

// dW[k,c] = sum_z part[z][k][c];  dcent[k,c] = - sum_n g[n,k,c] asum[n,k],  asum[n,k] = sum_s a[n,s,k]
__global__ void __launch_bounds__(256)
nv_bwd_reduce_kernel(const float* __restrict__ part, int splits, int C, int N, int S, int K,
                     const float* __restrict__ g, const float* __restrict__ assign,
                     float* __restrict__ dW, float* __restrict__ dcent) {
  __shared__ float asum_s[8];
  const int k = blockIdx.x;      // one block per cluster, K blocks
  // dW row
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float v = 0.f;
    for (int z = 0; z < splits; ++z) v += part[((long long)z * K + k) * C + c];
    dW[(long long)k * C + c] = v;
  }
  // dcent row: accumulate over images; asum[n,k] by a block reduction per image
  float* dc = dcent + (long long)k * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) dc[c] = 0.f;
  for (int n = 0; n < N; ++n) {
    float a = 0.f;
    for (int s = threadIdx.x; s < S; s += blockDim.x) a += __ldg(assign + ((long long)n * S + s) * K + k);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) asum_s[threadIdx.x >> 5] = a;
    __syncthreads();
    float tot = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += asum_s[i];
    const float* gn = g + ((long long)n * K + k) * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) dc[c] -= __ldg(gn + c) * tot;
  }
}

int launch_netvlad_backward(const float* x, bool nhwc, int N, int C, int S, const float* conv_w,
                            const float* centroids, int K, const float* g, bool normalize_input, float* assign,
                            float* invnorm, float* dz, float* part, int splits, float* dx, float* dW,
                            float* dcent, cudaStream_t s, uint64_t* launches) {
  IBL_REQUIRE(C % 4 == 0 && C <= 2048, "NetVLAD backward: C must be a multiple of 4 and <= 2048");
  IBL_REQUIRE(K >= 1 && K <= NB_K, "NetVLAD backward kernels serve 1..64 clusters");
  // recompute a and 1/|x| with the forward kernels (raw vlad goes to `part` as scratch and is discarded)
  FeatV f;
  f.p = x;
  f.sN = (long long)S * C;
  if (nhwc) { f.sS = C; f.sC = 1; } else { f.sS = 1; f.sC = S; }
  IBL_RET(launch_netvlad_assign(x, nhwc, N, C, S, conv_w, K, normalize_input, assign, invnorm, s));
  dim3 g1((unsigned)cdiv(S, 32), (unsigned)N);
  nv_bwd_dz_kernel<<<g1, 256, 0, s>>>(f, nhwc, C, S, K, g, centroids, assign, invnorm, dz);
  IBL_CUDA_OK(cudaGetLastError());
  const size_t smem = (size_t)(2 * 32 * 65 + 2 * 64 * 65 + 32 * (C + 1)) * sizeof(float);
  static DeviceOnce attr_done;   // the attribute is per device
  if (!attr_done.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(nv_bwd_dx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_done.mark();
  }
  const long long dN = (long long)S * C, dS = nhwc ? C : 1, dC = nhwc ? 1 : S;
  nv_bwd_dx_kernel<<<g1, 256, smem, s>>>(f, nhwc, C, S, K, g, conv_w, assign, dz, invnorm, normalize_input ? 1 : 0, dx,
                                         dN, dS, dC);
  IBL_CUDA_OK(cudaGetLastError());
  const long long R = (long long)N * S;
  int rows_per_split = (int)((R + splits - 1) / splits);
  rows_per_split = ((rows_per_split + 15) / 16) * 16;
  const int nsplit = (int)((R + rows_per_split - 1) / rows_per_split);
  nv_bwd_dw_kernel<<<dim3((unsigned)cdiv(C, 64), (unsigned)nsplit), 256, 0, s>>>(f, nhwc, C, S, N, K, dz, invnorm,
                                                                                  rows_per_split, part);
  IBL_CUDA_OK(cudaGetLastError());
  nv_bwd_reduce_kernel<<<K, 256, 0, s>>>(part, nsplit, C, N, S, K, g, assign, dW, dcent);
  IBL_CUDA_OK(cudaGetLastError());
  *launches += 5;
  return IBL_OK;
}

}  // namespace ibl
