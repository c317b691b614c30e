// Shared declarations for libiblb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>

#include "../../include/iblb200.h"

namespace ibl {

void set_last_error(const std::string& s);

#define IBL_CUDA_OK(expr)                                                          \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess) {                                                       \
      ::ibl::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e) +   \
                            " (" __FILE__ ":" + std::to_string(__LINE__) + ")");   \
      return IBL_ERR_CUDA;                                                         \
    }                                                                              \
  } while (0)

#define IBL_RET(expr)                 \
  do {                                \
    int _s = (expr);                  \
    if (_s != IBL_OK) return _s;      \
  } while (0)

#define IBL_REQUIRE(cond, msg)                                  \
  do {                                                          \
    if (!(cond)) {                                              \
      ::ibl::set_last_error(std::string("bad argument: ") + msg); \
      return IBL_ERR_BAD_ARG;                                   \
    }                                                           \
  } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// NetVLAD cluster counts the kernels serve: 1..64.  The tensor-core kernel pads K < 64 to 64 clusters; more than 64
// would need a different shared-memory plan there and a two-block softmax in the CUDA-core kernels.
constexpr int NETVLAD_MAX_K = 64;
static inline int check_netvlad_clusters(int K) {
  if (K < 1) {
    set_last_error("bad argument: NetVLAD num_clusters must be in 1..64, got " + std::to_string(K));
    return IBL_ERR_BAD_ARG;
  }
  if (K > NETVLAD_MAX_K) {
    set_last_error("unsupported: NetVLAD num_clusters must be in 1..64, got " + std::to_string(K));
    return IBL_ERR_UNSUPPORTED;
  }
  return IBL_OK;
}

// "Done once" flag per CUDA device: function attributes (cudaFuncSetAttribute) and device properties belong
// to a device, and one process may drive several GPUs (one engine each).  done()/mark() look at the calling
// thread's current device; setting an attribute twice from two threads is harmless, launching before it
// is set is not, so mark() comes after the setter.
struct DeviceOnce {
  std::atomic<unsigned long long> mask[4];
  DeviceOnce() { for (auto& m : mask) m.store(0); }
  static int cur() { int d = 0; cudaGetDevice(&d); return d & 255; }
  bool done() const { const int d = cur(); return (mask[d >> 6].load(std::memory_order_acquire) >> (d & 63)) & 1ull; }
  void mark() { const int d = cur(); mask[d >> 6].fetch_or(1ull << (d & 63), std::memory_order_release); }
};

// SM count of the calling thread's current device
static inline int device_sm_count() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  return sms;
}

// One conv layer of the VGG16 trunk.
struct ConvLayer {
  int cin, cout;
  bool relu;       // ReLU after the conv (all but conv5_3, vgg.py:41-42)
  bool pool;       // MaxPool2x2 after the ReLU (blocks 1-4)
};

// Device-side parameter store of one conv layer.
struct ConvParams {
  float* w_tck = nullptr;            // SIMT layout  [9][Cin][Cout] fp32
  float* bias = nullptr;             // [Cout]
  __nv_bfloat16* w_hi = nullptr;     // TC layout    [9][Cout][Cin_pad] bf16 (hi part)
  __nv_bfloat16* w_lo = nullptr;     //                                      (lo part)
  int cin_pad = 0;
};

// ---- launchers implemented in the .cu files ------------------------------------------------
// simt_conv.cu
int launch_repack_weights(const float* w_oihw, int cout, int cin, ConvParams& p, cudaStream_t s);
int launch_conv3x3_simt(const float* x_nhwc, const ConvParams& p, int N, int H, int W, int cin,
                        int cout, bool relu, float* y_nhwc, cudaStream_t s);
int launch_conv1_1(const float* x_nchw, const ConvParams& p, int N, int H, int W, float* y_nhwc, cudaStream_t s);
int launch_maxpool2x2(const float* x, int N, int H, int W, int C, float* y, cudaStream_t s);
int launch_nhwc_to_nchw(const float* x, int N, int S, int C, float* y, cudaStream_t s);
int launch_u8_hwc_to_nchw_norm(const uint8_t* x, int N, int H, int W, const float* mean, const float* stdv, float* y,
                               cudaStream_t s);
int launch_global_maxpool_nhwc(const float* x, int N, int S, int C, float* y, cudaStream_t s);
int launch_planes_to_f32(const __nv_bfloat16* hi, const __nv_bfloat16* lo, size_t n, float* y,
                         cudaStream_t s);
int launch_f32_to_planes(const float* x, size_t n, __nv_bfloat16* hi, __nv_bfloat16* lo,
                         cudaStream_t s);

// tc_conv.cu  (wgmma + TMA implicit GEMM, bf16 hi/lo split operands)
struct TcConvPlan;   // opaque per-engine cache of TMA descriptors
int tc_driver_init();   // resolves cuTensorMapEncodeTiled; IBL_ERR_NO_DEVICE if unavailable
int launch_conv3x3_tc(const __nv_bfloat16* x_hi, const __nv_bfloat16* x_lo, const ConvParams& p,
                      int N, int H, int W, int cin, int cout, bool relu, bool pool,
                      __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, float* y_f32, cudaStream_t s,
                      float* ssq = nullptr, int* ssq_parts = nullptr);
int launch_conv1_fused_tc(const float* x_nchw, const float* w1_oihw, const float* bias1, const ConvParams& p2, int N, int H,
                          int W, __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, cudaStream_t s);
int launch_maxpool2x2_planes(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int N, int H, int W,
                             int C, __nv_bfloat16* yhi, __nv_bfloat16* ylo, cudaStream_t s);
int tc_selftest(float* max_rel_err, cudaStream_t s);
// sort_rows.cu  (full argsort of distance-matrix rows: the training samplers' mining)
int launch_argsort_rows(const float* dist, long long ld, int m, int n, long long* idx, unsigned long long* scratch,
                        cudaStream_t s, uint64_t* launches);
// resize.cu  (Pillow-exact 8-bit bilinear resample)
int launch_resize_bilinear_u8(const uint8_t* x, int N, int Hin, int Win, int Hout, int Wout, const int* bounds_h,
                              const int* kk_h, int ksize_h, const int* bounds_v, const int* kk_v, int ksize_v,
                              uint8_t* tmp, uint8_t* out, cudaStream_t s, uint64_t* launches);
// jpeg.cu  (baseline and progressive JPEG decode, bit-exact with libjpeg's defaults; the parser is host code)
// Per-engine decode workspace (the JPEG and PNG paths each own one): pinned staging blob, its device copy, and an
// arena for tables, coefficients, planes or inflated rows.  `copied` marks the end of the last H2D copy from `host`.
struct JpegWs {
  uint8_t* host = nullptr;
  size_t host_cap = 0;
  void* blob = nullptr;
  size_t blob_cap = 0;
  void* arena = nullptr;
  size_t arena_cap = 0;
  cudaEvent_t copied = nullptr;
  bool pending = false;
};
void jpeg_ws_destroy(JpegWs* ws);
int ws_open(JpegWs** pws);
int grow_device(void** p, size_t* cap, size_t need);   // device buffer of at least `need` bytes (contents dropped)
int stage_host(JpegWs* ws, size_t bytes);             // pinned staging once the previous H2D copy no longer reads it
int jpeg_decode_u8(JpegWs** ws, const uint8_t* const* files, const size_t* lens, int N, uint8_t* out_u8,
                   const uint64_t* out_offsets, int* status, int* err_dev, cudaStream_t s, uint64_t* launches);
int jpeg_decode_progressive_u8(JpegWs** ws, const uint8_t* const* files, const size_t* lens, int N, uint8_t* out_u8,
                               const uint64_t* out_offsets, int* status, int* err_dev, cudaStream_t s,
                               uint64_t* launches);
// png.cu  (8-bit non-interlaced PNG decode, bit-exact with Pillow; the chunk parse is host code)
int png_decode_u8(JpegWs** ws, const uint8_t* const* files, const size_t* lens, int N, uint8_t* out_u8,
                  const uint64_t* out_offsets, int* status, int* err_dev, cudaStream_t s, uint64_t* launches);
// color_jitter.cu  (T.ColorJitter, bit-exact with torchvision's PIL path)
struct JitterWs;   // opaque per-engine workspace: pinned staging of descriptors, device copy, L sums
void jitter_ws_destroy(JitterWs* ws);
int color_jitter_u8(JitterWs** ws, uint8_t* buf, const uint64_t* out_offsets, const int* H, const int* W,
                    const ibl_color_jitter_params* params, int N, cudaStream_t s, uint64_t* launches);
// tc_conv_bwd.cu  (dgrad filter re-layout, wgmma wgrad, ReLU mask, pool backward, conv1_1 wgrad)
int launch_repack_weights_dgrad(const float* w_tck, int cout, int cin, __nv_bfloat16* w_hi, __nv_bfloat16* w_lo,
                                cudaStream_t s);
int launch_relu_mask_planes(const float* g, const float* y, size_t n, bool relu, __nv_bfloat16* hi, __nv_bfloat16* lo,
                            cudaStream_t s);
int launch_maxpool2x2_bwd(const float* x, const float* gy, int N, int H, int W, int C, float* gx, cudaStream_t s);
int wgrad_tc_splits(int N, int H, int W, int cin, int cout);
int launch_conv_wgrad_tc(const __nv_bfloat16* g_hi, const __nv_bfloat16* g_lo, const __nv_bfloat16* x_hi,
                         const __nv_bfloat16* x_lo, int N, int H, int W, int cin, int cout, float* part, int splits,
                         float* bpart, float* dw_oihw, float* db, cudaStream_t s);
int launch_conv1_1_wgrad(const float* x_nchw, const __nv_bfloat16* g_hi, const __nv_bfloat16* g_lo, int N, int H, int W,
                         float* part, float* dw_oihw, float* db, cudaStream_t s);
// tc_conv1.cu
int launch_conv1_1_tc(const float* x_nchw, const float* w_oihw, const float* bias, int N, int H, int W,
                      __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, cudaStream_t s);
// tc_probe.cu
int debug_gmma_strided(const void* A, int rows, const void* B, int s0, int group_rows, int half_rows, int base_mode,
                       float* D, cudaStream_t s);
int debug_wgmma_rs_halo(const void* W, const void* X, int pitch, int hrows, int n, int s0, float* D, cudaStream_t s);
// tc_netvlad.cu
int debug_gemm_tn(const float* A, const float* B, float* C, cudaStream_t s);
int netvlad_tc_units(int B, int S);
int launch_netvlad_tc(const __nv_bfloat16* x_hi, const __nv_bfloat16* x_lo, int B, int S, int K,
                      const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo, const float* ssq, int ssq_parts,
                      const float* cent, bool normalize_input, float* part, float* asum_part, int* ticket,
                      float* vlad_raw, float* vlad_norm, cudaStream_t s);
int launch_global_maxpool_planes(const __nv_bfloat16* hi, const __nv_bfloat16* lo, int N, int S, int C, float* y,
                                 cudaStream_t s);

// tc_gemm.cu  (wgmma NT GEMM on bf16 hi/lo planes: distance/top-16, dense distance, PCA partials)
int dist_top16_max_runs(int n_valid);
int launch_dist_top16_tc(const __nv_bfloat16* q_hi, const __nv_bfloat16* q_lo, const float* qn, int m,
                         const __nv_bfloat16* d_hi, const __nv_bfloat16* d_lo, const float* dn, int n,
                         int n_valid, int K, float* cand_d, long long* cand_i, int max_runs, int* runs_out,
                         cudaStream_t s);
int launch_dist_dense_tc(const __nv_bfloat16* q_hi, const __nv_bfloat16* q_lo, const float* qn, int m,
                         const __nv_bfloat16* d_hi, const __nv_bfloat16* d_lo, const float* dn, int n, int K,
                         float* out, long long ld_out, cudaStream_t s);
// tc_dist1.cu  (fp16 screening + exact re-scoring + guard + exact fallback) on a database prepared by
// launch_db_prepare (plane, aux, maxima as rows_f16_kernel / dist_colmax_kernel make them): the single-pass screening
// and the small-batch streaming search
int launch_db_prepare(const float* db, int n, int d, __half* plane, float4* aux, float* dbmax, cudaStream_t s);
size_t dist1_workspace_bytes(int m, int d, size_t* off /*[7]*/);
const int* dist1_flag_counter(const void* ws, int m, int d);
int launch_dist_topk_1pass_prepared(const float* q, int m, const float* db, const __half* plane, const float4* aux,
                                    const float* dbmax, int n, int d, int k, long long idx_base, void* ws,
                                    float* out_dist, long long* out_idx, uint64_t* launches, cudaStream_t s);
size_t db_scan_workspace_bytes(int m, int n, int d);
int launch_db_scan_topk(const float* q, int m, const float* db, const __half* plane, const float4* aux,
                        const float* dbmax, int n, int d, int k, long long idx_base, void* ws, float* out_dist,
                        long long* out_idx, uint64_t* launches, cudaStream_t s);
const int* db_scan_flag_counter(const void* ws, int m, int n, int d);
// ... and the same guard + exact fallback after the bf16x3 screening of tc_gemm.cu
size_t dist_guard_workspace_bytes(int m);
int launch_dist_guard_bf16x3(const float* q, const float* q_sq, const float2* q_err, int m, const float* db,
                             const float* db_sq, const float2* db_err, int n_valid, int d, const float* screened, int kc,
                             int k, long long idx_base, void* ws, float* out_dist, long long* out_idx,
                             uint64_t* launches, cudaStream_t s);
// out3 (zeroed by the caller) = max over the n rows of {|lo|, |x - hi - lo|, |x|^2} (launch_planes_sqnorm's err, sq)
int launch_bf16x3_colmax(const float2* err, const float* sq, int n, float* out3, cudaStream_t s);
int pca_tc_splits(int P, int D);
int launch_pca_partial_tc(const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo, int P,
                          const __nv_bfloat16* v_hi, const __nv_bfloat16* v_lo, int N, int D,
                          float* partial, int* splits_out, cudaStream_t s);
int launch_rescore_sort(const float* q, const float* qn, int m, const float* db, const float* dbn, int d,
                        const long long* cand_i, int kc, int k_out, long long idx_base, float* out_dist,
                        long long* out_idx, cudaStream_t s, int sq_stride = 1);
// out = bias + sum of the partials, then L2 per row when `normalize` (false: the pre-normalisation y of training)
int launch_pca_finalize(const float* partial, int splits, int N, int P, const float* bias, float* out,
                        cudaStream_t s, bool normalize = true);
// tc_pca_bwd.cu: backward of the PCA layer (gy planes [N][Pp], Pp = P rounded up to 8)
int launch_pca_gy_planes(const float* gy, int N, int P, int Pp, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t s);
int launch_pca_dgrad_tc(const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo, int P, int D, const __nv_bfloat16* g_hi,
                        const __nv_bfloat16* g_lo, int Pp, int N, float* gv, cudaStream_t s);
int launch_pca_wgrad_tc(const __nv_bfloat16* v_hi, const __nv_bfloat16* v_lo, int N, int D, const __nv_bfloat16* g_hi,
                        const __nv_bfloat16* g_lo, int P, int Pp, float* gW, cudaStream_t s);
int launch_pca_bias_grad(const float* gy, int N, int P, float* gb, cudaStream_t s);
int launch_pca_tn_simt(const float* A, long long sr, long long sk, int R, int K, const float* B, int D, float* C,
                       cudaStream_t s);

// netvlad.cu
struct NetvladWorkspace {
  float* assign = nullptr;   // [N,S,K]  soft-assignment * inv-norm handled in kernel
  float* invnorm = nullptr;  // [N,S]
  float* asum = nullptr;     // [N,K]
  float* raw = nullptr;      // [N,K,C]  (used when the caller does not want vlad_raw)
  size_t cap_N = 0;
  int cap_S = 0, cap_K = 0, cap_C = 0;
};
int launch_netvlad(const float* feat, bool nhwc, int N, int C, int S, const float* conv_w,
                   const float* centroids, int K, bool normalize_input, float* assign,
                   float* invnorm, float* asum, float* vlad_raw, float* vlad_norm,
                   cudaStream_t s, uint64_t* launches);
int launch_vlad_normalize(const float* raw, int N, int K, int C, float* out, cudaStream_t s);
int launch_netvlad_assign(const float* feat, bool nhwc, int N, int C, int S, const float* conv_w, int K,
                          bool normalize_input, float* assign, float* invnorm, cudaStream_t s);
// netvlad_bwd.cu
int launch_netvlad_backward(const float* x, bool nhwc, int N, int C, int S, const float* conv_w,
                            const float* centroids, int K, const float* g, bool normalize_input, float* assign,
                            float* invnorm, float* dz, float* part, int splits, float* dx, float* dW,
                            float* dcent, cudaStream_t s, uint64_t* launches);

// gemm_simt.cu  (C = A[m,K] . B[n,K]^T family)
int launch_pca_l2(const float* v, int N, int D, const float* W, const float* b, int P,
                  float* partial, int splits, float* out, cudaStream_t s, uint64_t* launches, bool normalize = true);
int launch_l2_normalize_rows(const float* x, int N, int D, float* out, cudaStream_t s);
int launch_row_sqnorm(const float* x, int N, int D, float* out, cudaStream_t s);
int launch_scale(const float* x, float s, int n, float* y, cudaStream_t st);
int launch_planes_sqnorm(const float* x, int N, int D, __nv_bfloat16* hi, __nv_bfloat16* lo, float* sq,
                         float2* err, cudaStream_t st);   // err (may be null): per row {|lo|, |x - hi - lo|}
int launch_l2dist_dense(const float* q, const float* qn, int m, const float* db, const float* dbn,
                        int n, int d, float* out, long long ld_out, cudaStream_t s);

// rerank.cu  (k-reciprocal re-ranking: exact neighbour pass + sparse stage)
size_t knn_rowmax_workspace_bytes(int N, int d, int n_rows, int w);
const int* knn_rowmax_flag_counter(const void* ws, int N, int d, int n_rows, int w);
int launch_knn_rowmax(const float* X, int N, int d, int row0, int n_rows, int w, void* ws, long long* out_idx,
                      float* out_dist, float* out_max, uint64_t* launches, cudaStream_t s);
struct RerankWs;
RerankWs* rerank_ws_create();
void rerank_ws_destroy(RerankWs* w);
size_t rerank_ws_bytes(const RerankWs* w);
int launch_rerank_topk(RerankWs* W, const float* X, int N, int m, int d, const long long* nbr, const float* nbr_dist,
                       int w, const float* rowmax, int k1, int k2, float lam, const long long* orig, int k_orig, int k,
                       float* out_dist, long long* out_idx, uint64_t* launches, cudaStream_t s);
int launch_rerank_dense(RerankWs* W, const float* qg, const float* qq, const float* gg, int m, int n, int k1, int k2,
                        double lam, float* out, uint64_t* launches, cudaStream_t s);

// topk.cu
int launch_topk_rows(const float* dist, long long ld, int m, int n_valid, int k, int64_t idx_base,
                     float* out_dist, int64_t* out_idx, bool accumulate, cudaStream_t s);
int launch_topk_rows_seg(const float* dist, long long ld, int m, int n_valid, int k, int segs, int seg,
                         int64_t idx_base, float* out_dist, int64_t* out_idx, cudaStream_t s);
int launch_topk_merge(const float* cand_dist, const int64_t* cand_idx, int parts, int m, int k_in,
                      int k_out, float* out_dist, int64_t* out_idx, cudaStream_t s);

}  // namespace ibl
