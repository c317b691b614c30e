// Baseline JPEG decode on the GPU, bit-identical to Pillow's `Image.open(f).convert('RGB')` (Preprocessor.__getitem__,
// ibl/utils/data/preprocessor.py:31-42), which runs libjpeg(-turbo) with its defaults: accurate integer IDCT
// (JDCT_ISLOW, jidctint.c), "fancy" triangular upsampling (jdsample.c) and the integer YCbCr->RGB tables (jdcolor.c).
//
// Host: `parse_jpeg` reads the markers, builds libjpeg's derived Huffman tables (jdhuff.c jpeg_make_d_derived_tbl,
// including its validity checks), splits the entropy-coded data at RSTn and removes the stuffed 0x00 after 0xFF.
// Everything the parser does not accept is left to the caller (Pillow on the host).
//
// Device, per batch (all on the caller's stream, one pinned H2D copy of tables + destuffed entropy data):
//   1. jpeg_sync_kernel     every restart interval is cut into runs of kRunBits bits.  A run's decoder starts at
//                           "coefficient 0 of the MCU's first block" at the run's first bit (the first run of an
//                           interval starts in its known state) and decodes codewords until it passes the run's end;
//                           it records the state (bit position, block within the MCU, zig-zag index) at the first
//                           codeword boundary at or past that end.  Baseline Huffman streams self-synchronise, so a
//                           run started at a wrong boundary usually falls onto the true codeword boundaries within a
//                           few codewords (Weissenberger & Schmidt, "Massively parallel Huffman decoding on GPUs",
//                           ICPP 2018).
//   2. jpeg_fix_kernel      one block per image: every run is decoded again from its predecessor's end state; a run
//                           whose end state changes marks its successor for another pass, until no state changes.
//                           The fixed point is the sequential decode whatever happens in between: after pass k the
//                           first k runs of every interval are exact, so the worst case is sequential propagation.
//                           Invalid codes met from a wrong start end the run in an "invalid" state and never fault.
//                           Then an exclusive scan of the runs' completed-block counts gives each run's first block.
//   3. jpeg_write_kernel    every run decodes once more from its exact start state and writes its coefficients,
//                           natural order, into a zeroed int16 [blocks][64] buffer (the DC entry holds the coded DC
//                           difference); an invalid code on the true path, or an interval that ends before its last
//                           block, sets the image's error word.
//   4. jpeg_dc_kernel       DC differences are prefix-summed per component in MCU order, restarting at every interval.
//   5. jpeg_idct_kernel     dequantise + jpeg_idct_islow per block into component planes at libjpeg's sizes.
//   6. jpeg_color_kernel    fancy upsampling (h2v1 / h2v2, edge replication) + YCbCr->RGB, uint8 HWC out.
// Every bit fetch reads at most 5 bytes from a position inside its interval, and every interval is followed by 8 zero
// bytes in the staging buffer: no input, however corrupt, reads or writes outside the buffers.
//
// Progressive files (SOF2): `parse_jpeg(..., progressive=true)` records the scan script, and the jpeg_prog_*_kernel
// family decodes the scans of every image in file order into the same coefficient buffer (frame MCU order), after
// which steps 5 and 6 run unchanged.
#include <string.h>

#include <algorithm>
#include <new>
#include <vector>

#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace ibl {

namespace {

constexpr int kRunBits = 1024;        // bits per decoder run (subsequence)
constexpr int kLookBits = 9;          // Huffman lookahead bits
constexpr int kFixThreads = 512;
constexpr int kDcThreads = 256;
constexpr uint64_t kInvalid = 1ull << 63;
constexpr int kPad = 8;               // zero bytes after every interval
constexpr int kProgWarps = 4;         // warps per block of the sequential progressive scan kernels

// jpeg_natural_order (jutils.c): zig-zag index -> natural (row-major) index
__constant__ uint8_t c_natural[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
const uint8_t h_natural[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// libjpeg's derived decoding table (jdhuff.c d_derived_tbl) plus a kLookBits lookahead
struct HuffTab {
  int32_t maxcode[18];              // largest code of length l, -1 if none
  int32_t valoff[17];               // huffval index of a code of length l = valoff[l] + code
  uint16_t look[1 << kLookBits];    // (length << 8) | symbol for codes of <= kLookBits bits, 0 otherwise
  uint8_t huffval[256];
};

struct ImgDev {
  int width, height, ncomp;
  int mcus_x, mcus_y, bpm;          // MCU grid, blocks per MCU
  int8_t blk_comp[6], blk_dx[6], blk_dy[6];
  int comp_hs[3], comp_vs[3];       // sampling factors (1x1 for a single-component scan)
  int comp_w[3], comp_h[3];         // libjpeg's downsampled_width / downsampled_height
  int plane_w[3];                   // padded plane rows: blocks across * 8
  uint64_t plane_off[3];            // byte offsets in the plane arena
  uint64_t coef_block;              // first block in the coefficient arena
  uint64_t out_off;                 // byte offset in the caller's output
  int nblocks;
  int first_seq, n_seq;
  uint16_t q[3][64];                // quantisation table per component, natural order
};

struct IntervalDev {
  uint64_t byte_base;               // first byte in the entropy arena
  uint32_t nbits;
  int img;                          // index into the ImgDev array
  int first_block;                  // first block of the interval within its image
  int nblocks;
  int first_seq, n_seq;
};

struct Cursor {
  uint32_t pos;
  int blk, zz;
};

__host__ __device__ inline uint64_t pack(const Cursor& c) {
  return (uint64_t)c.pos | ((uint64_t)c.blk << 32) | ((uint64_t)c.zz << 40);
}
__host__ __device__ inline Cursor unpack(uint64_t v) {
  return Cursor{(uint32_t)v, (int)((v >> 32) & 255), (int)((v >> 40) & 255)};
}

// 32 bits starting at bit `pos` (MSB first); reads bytes pos/8 .. pos/8 + 4
__host__ __device__ inline uint32_t peek32(const uint8_t* d, uint32_t pos) {
  const uint8_t* p = d + (pos >> 3);
  const uint64_t v = ((uint64_t)p[0] << 32) | ((uint64_t)p[1] << 24) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 8) |
                     (uint64_t)p[4];
  return (uint32_t)(v >> (8 - (pos & 7)));
}

__host__ __device__ inline int huff_decode(const HuffTab& t, uint32_t bits, int* len) {
  const uint32_t e = t.look[bits >> (32 - kLookBits)];
  if (e) {
    *len = (int)(e >> 8);
    return (int)(e & 255);
  }
  for (int l = kLookBits + 1; l <= 16; ++l) {
    const int32_t code = (int32_t)(bits >> (32 - l));
    if (code <= t.maxcode[l]) {
      *len = l;
      return t.huffval[(t.valoff[l] + code) & 255];
    }
  }
  return -1;
}

// HUFF_EXTEND (jdhuff.h)
__host__ __device__ inline int extend(uint32_t v, int s) {
  return (int)v < (1 << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v;
}

// Decode codewords from `c` while c.pos < stop.  emit(blocks_done, zz, value) is called for the DC difference
// (zz 0) and every nonzero AC coefficient; blocks_done counts the blocks completed since the start.  Mirrors
// jdhuff.c decode_mcu: a nonzero coefficient past zig-zag index 63 lands on index 63 (jpeg_natural_order's guard
// entries), a block ends at EOB or once the index passes 63.  Returns false at an invalid code.
template <class Emit>
__host__ __device__ inline bool decode_run(const uint8_t* d, uint32_t stop, const HuffTab* tabs, const int8_t* blk_comp,
                                           int bpm, Cursor& c, int& done, Emit emit) {
  while (c.pos < stop) {
    const uint32_t bits = peek32(d, c.pos);
    const int comp = blk_comp[c.blk];
    int len;
    if (c.zz == 0) {
      const int s = huff_decode(tabs[2 * comp], bits, &len);
      if (s < 0) return false;
      emit(done, 0, s ? extend((bits << len) >> (32 - s), s) : 0);
      c.pos += len + s;
      c.zz = 1;
    } else {
      const int rs = huff_decode(tabs[2 * comp + 1], bits, &len);
      if (rs < 0) return false;
      const int r = rs >> 4, s = rs & 15;
      if (s) {
        c.zz += r;
        emit(done, c.zz, extend((bits << len) >> (32 - s), s));
        c.zz += 1;
        c.pos += len + s;
      } else {
        c.zz = (r == 15) ? c.zz + 16 : 64;
        c.pos += len;
      }
    }
    if (c.zz >= 64) {
      c.zz = 0;
      if (++c.blk == bpm) c.blk = 0;
      ++done;
    }
  }
  return true;
}

struct NoEmit {
  __host__ __device__ void operator()(int, int, int) const {}
};

struct Batch {
  const ImgDev* img;
  const IntervalDev* iv;
  const HuffTab* tabs;              // [images][3 components][DC, AC]
  const int* seq_iv;                // run -> interval
  const uint8_t* bytes;             // entropy arena
  int n_seq;
  uint64_t* st;                     // end state of every run
  uint64_t* st_new;
  int* cnt;                         // blocks completed within every run
  int* cnt_new;
  int* first_blk;                   // blocks completed in the interval before the run's start
  uint8_t* need;
  uint8_t* chg;
  int16_t* coef;
  uint8_t* planes;
  uint8_t* out;
  int* err;
  const int* err_slot;              // ImgDev index -> caller's image index
};

__device__ inline uint32_t run_stop(const IntervalDev& iv, int j) {
  const uint64_t e = (uint64_t)(j + 1) * kRunBits;
  return e < iv.nbits ? (uint32_t)e : iv.nbits;
}

__global__ void jpeg_sync_kernel(Batch b) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < b.n_seq; s += gridDim.x * blockDim.x) {
    const IntervalDev iv = b.iv[b.seq_iv[s]];
    const ImgDev& im = b.img[iv.img];
    const int j = s - iv.first_seq;
    Cursor c{(uint32_t)j * kRunBits, 0, 0};
    int done = 0;
    const bool ok = decode_run(b.bytes + iv.byte_base, run_stop(iv, j), b.tabs + 6 * iv.img, im.blk_comp, im.bpm, c,
                               done, NoEmit());
    b.st[s] = ok ? pack(c) : kInvalid;
    b.cnt[s] = done;
  }
}

__device__ inline Cursor start_of(const Batch& b, int s, int j) {
  if (j == 0) return Cursor{0, 0, 0};
  const uint64_t p = b.st[s - 1];
  return p == kInvalid ? Cursor{(uint32_t)j * kRunBits, 0, 0} : unpack(p);
}

__global__ void __launch_bounds__(kFixThreads) jpeg_fix_kernel(Batch b) {
  const ImgDev& im = b.img[blockIdx.x];
  const int s0 = im.first_seq, ns = im.n_seq;
  const HuffTab* tabs = b.tabs + 6 * blockIdx.x;
  for (int s = s0 + threadIdx.x; s < s0 + ns; s += kFixThreads) b.need[s] = s != b.iv[b.seq_iv[s]].first_seq;
  __syncthreads();
  for (;;) {
    for (int s = s0 + threadIdx.x; s < s0 + ns; s += kFixThreads) {
      if (!b.need[s]) continue;
      const IntervalDev& iv = b.iv[b.seq_iv[s]];
      const int j = s - iv.first_seq;
      Cursor c = start_of(b, s, j);
      int done = 0;
      const bool ok = decode_run(b.bytes + iv.byte_base, run_stop(iv, j), tabs, im.blk_comp, im.bpm, c, done, NoEmit());
      b.st_new[s] = ok ? pack(c) : kInvalid;
      b.cnt_new[s] = done;
    }
    __syncthreads();
    int changed = 0;
    for (int s = s0 + threadIdx.x; s < s0 + ns; s += kFixThreads) {
      uint8_t ch = 0;
      if (b.need[s]) {
        b.cnt[s] = b.cnt_new[s];
        if (b.st_new[s] != b.st[s]) {
          b.st[s] = b.st_new[s];
          ch = 1;
        }
      }
      b.chg[s] = ch;
      changed |= ch;
    }
    if (!__syncthreads_or(changed)) break;
    for (int s = s0 + threadIdx.x; s < s0 + ns; s += kFixThreads)
      b.need[s] = s != b.iv[b.seq_iv[s]].first_seq && b.chg[s - 1];
    __syncthreads();
  }
  // first block of every run: exclusive scan over the image, rebased to each interval's first run
  using Scan = cub::BlockScan<int, kFixThreads>;
  __shared__ typename Scan::TempStorage tmp;
  int carry = 0;
  for (int base = 0; base < ns; base += kFixThreads) {
    const int s = s0 + base + threadIdx.x;
    const int v = base + (int)threadIdx.x < ns ? b.cnt[s] : 0;
    int ex, tot;
    Scan(tmp).ExclusiveSum(v, ex, tot);
    if (base + (int)threadIdx.x < ns) b.cnt_new[s] = carry + ex;
    carry += tot;
    __syncthreads();
  }
  for (int s = s0 + threadIdx.x; s < s0 + ns; s += kFixThreads)
    b.first_blk[s] = b.cnt_new[s] - b.cnt_new[b.iv[b.seq_iv[s]].first_seq];
}

__global__ void jpeg_write_kernel(Batch b) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < b.n_seq; s += gridDim.x * blockDim.x) {
    const IntervalDev iv = b.iv[b.seq_iv[s]];
    const ImgDev& im = b.img[iv.img];
    const int j = s - iv.first_seq;
    const int first = b.first_blk[s];
    int* err = b.err + b.err_slot[iv.img];
    if (j > 0 && b.st[s - 1] == kInvalid) {           // the true path hit an invalid code in an earlier run
      if (first < iv.nblocks) atomicOr(err, 1);
      continue;
    }
    Cursor c = start_of(b, s, j);
    int done = 0;
    int16_t* coef = b.coef + (im.coef_block + (uint64_t)iv.first_block) * 64;
    const int limit = iv.nblocks;
    auto emit = [&](int k, int zz, int v) {
      const int blk = first + k;
      if (blk < limit) coef[(uint64_t)blk * 64 + c_natural[zz < 63 ? zz : 63]] = (int16_t)v;
    };
    const bool ok = decode_run(b.bytes + iv.byte_base, run_stop(iv, j), b.tabs + 6 * iv.img, im.blk_comp, im.bpm, c,
                               done, emit);
    if (first + done < limit && (!ok || j == iv.n_seq - 1)) atomicOr(err, ok ? 2 : 1);
  }
}

// DC prediction (jdhuff.c: last_dc_val per component, reset at every restart): int accumulation, stored as JCOEF
__global__ void __launch_bounds__(kDcThreads) jpeg_dc_kernel(Batch b) {
  const IntervalDev& iv = b.iv[blockIdx.x];
  const ImgDev& im = b.img[iv.img];
  int16_t* coef = b.coef + (im.coef_block + (uint64_t)iv.first_block) * 64;
  using Scan = cub::BlockScan<int, kDcThreads>;
  __shared__ typename Scan::TempStorage tmp;
  int carry[3] = {0, 0, 0};
  for (int base = 0; base < iv.nblocks; base += kDcThreads) {
    const int k = base + threadIdx.x;
    const int comp = k < iv.nblocks ? im.blk_comp[k % im.bpm] : -1;
    const int v = comp >= 0 ? coef[(uint64_t)k * 64] : 0;
    for (int ci = 0; ci < im.ncomp; ++ci) {
      int inc, tot;
      Scan(tmp).InclusiveSum(comp == ci ? v : 0, inc, tot);
      if (comp == ci) coef[(uint64_t)k * 64] = (int16_t)(carry[ci] + inc);
      carry[ci] += tot;
      __syncthreads();
    }
  }
}

// jidctint.c jpeg_idct_islow: CONST_BITS 13, PASS1_BITS 2, columns then rows, DESCALE with rounding, and the
// post-IDCT range limit (sample_range_limit + CENTERJSAMPLE indexed with & RANGE_MASK).
constexpr int kConstBits = 13, kPass1Bits = 2;
#define JFIX_0_298631336 2446
#define JFIX_0_390180644 3196
#define JFIX_0_541196100 4433
#define JFIX_0_765366865 6270
#define JFIX_0_899976223 7373
#define JFIX_1_175875602 9633
#define JFIX_1_501321110 12299
#define JFIX_1_847759065 15137
#define JFIX_1_961570560 16069
#define JFIX_2_053119869 16819
#define JFIX_2_562915447 20995
#define JFIX_3_072711026 25172

__host__ __device__ inline int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

__host__ __device__ inline uint8_t idct_range_limit(int x) {
  const int t = ((x & 1023) ^ 512) - 512;           // x & RANGE_MASK as a signed offset from CENTERJSAMPLE
  const int v = t + 128;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// one 1-D pass: in[0..7] at stride `is` -> out[0..7] at stride `os`, descaled by `shift`
template <class In, class Out>
__host__ __device__ inline void idct_1d(In in, Out out, int shift) {
  int z2 = in(2), z3 = in(6);
  int z1 = (z2 + z3) * JFIX_0_541196100;
  int tmp2 = z1 + z3 * (-JFIX_1_847759065);
  int tmp3 = z1 + z2 * JFIX_0_765366865;
  z2 = in(0);
  z3 = in(4);
  int tmp0 = (z2 + z3) * (1 << kConstBits);
  int tmp1 = (z2 - z3) * (1 << kConstBits);
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  tmp0 = in(7);
  tmp1 = in(5);
  tmp2 = in(3);
  tmp3 = in(1);
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  int z4 = tmp1 + tmp3;
  const int z5 = (z3 + z4) * JFIX_1_175875602;
  tmp0 *= JFIX_0_298631336;
  tmp1 *= JFIX_2_053119869;
  tmp2 *= JFIX_3_072711026;
  tmp3 *= JFIX_1_501321110;
  z1 *= -JFIX_0_899976223;
  z2 *= -JFIX_2_562915447;
  z3 *= -JFIX_1_961570560;
  z4 *= -JFIX_0_390180644;
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  out(0, descale(tmp10 + tmp3, shift));
  out(7, descale(tmp10 - tmp3, shift));
  out(1, descale(tmp11 + tmp2, shift));
  out(6, descale(tmp11 - tmp2, shift));
  out(2, descale(tmp12 + tmp1, shift));
  out(5, descale(tmp12 - tmp1, shift));
  out(3, descale(tmp13 + tmp0, shift));
  out(4, descale(tmp13 - tmp0, shift));
}

// coef (natural order) x q -> 8x8 samples at dst with row stride `ld`
__host__ __device__ inline void idct_islow(const int16_t* coef, const uint16_t* q, uint8_t* dst, int ld) {
  int ws[64];
#pragma unroll
  for (int c = 0; c < 8; ++c)
    idct_1d([&](int r) { return (int)coef[8 * r + c] * (int)q[8 * r + c]; },
            [&](int r, int v) { ws[8 * r + c] = v; }, kConstBits - kPass1Bits);
#pragma unroll
  for (int r = 0; r < 8; ++r)
    idct_1d([&](int c) { return ws[8 * r + c]; },
            [&](int c, int v) { dst[(size_t)r * ld + c] = idct_range_limit(v); }, kConstBits + kPass1Bits + 3);
}

// block k of image `im` (MCU order) -> its 8x8 samples in the component plane
__host__ __device__ inline void idct_block(const ImgDev& im, const int16_t* coef, uint8_t* planes, int k) {
  const int mcu = k / im.bpm, kb = k - mcu * im.bpm;
  const int comp = im.blk_comp[kb];
  const int bx = (mcu % im.mcus_x) * im.comp_hs[comp] + im.blk_dx[kb];
  const int by = (mcu / im.mcus_x) * im.comp_vs[comp] + im.blk_dy[kb];
  const int ld = im.plane_w[comp];
  alignas(16) int16_t c[64];
  const int4* src = reinterpret_cast<const int4*>(coef + (im.coef_block + k) * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) reinterpret_cast<int4*>(c)[i] = src[i];
  idct_islow(c, im.q[comp], planes + im.plane_off[comp] + (size_t)by * 8 * ld + (size_t)bx * 8, ld);
}

__global__ void jpeg_idct_kernel(Batch b) {
  const ImgDev& im = b.img[blockIdx.y];
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < im.nblocks; k += gridDim.x * blockDim.x)
    idct_block(im, b.coef, b.planes, k);
}

// jdsample.c: h2v1_fancy_upsample / h2v2_fancy_upsample for components at least 3 samples wide, box replication
// (h2v1_upsample / h2v2_upsample) otherwise; rows above the first and below the last replicate the edge row
// (jdmainct.c context rows), columns likewise (the special-cased first and last columns).
__host__ __device__ inline int chroma_at(const uint8_t* p, int ld, int cw, int ch, int hs, int vs, int x, int y) {
  if (hs == 1) return p[(size_t)y * ld + x];
  const int cx = x >> 1;
  if (vs == 1) {
    const uint8_t* row = p + (size_t)y * ld;
    if (cw <= 2) return row[cx];
    const int v3 = 3 * row[cx];
    return (x & 1) ? (v3 + row[cx + 1 < cw ? cx + 1 : cw - 1] + 2) >> 2 : (v3 + row[cx > 0 ? cx - 1 : 0] + 1) >> 2;
  }
  const int cy = y >> 1;
  const uint8_t* r0 = p + (size_t)cy * ld;
  if (cw <= 2) return r0[cx];
  const uint8_t* r1 = p + (size_t)((y & 1) ? (cy + 1 < ch ? cy + 1 : ch - 1) : (cy > 0 ? cy - 1 : 0)) * ld;
  auto colsum = [&](int i) { return 3 * r0[i] + r1[i]; };
  const int t = 3 * colsum(cx);
  return (x & 1) ? (t + colsum(cx + 1 < cw ? cx + 1 : cw - 1) + 7) >> 4 : (t + colsum(cx > 0 ? cx - 1 : 0) + 8) >> 4;
}

__host__ __device__ inline uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// jdcolor.c ycc_rgb_convert (SCALEBITS 16, FIX(x) = x * 65536 + 0.5) of pixel (x, y); grayscale is replicated
__host__ __device__ inline void color_pixel(const ImgDev& im, const uint8_t* planes, int x, int y, uint8_t* o) {
  const int Y = planes[im.plane_off[0] + (size_t)y * im.plane_w[0] + x];
  if (im.ncomp == 1) {
    o[0] = o[1] = o[2] = (uint8_t)Y;
    return;
  }
  const int hs = im.comp_hs[0], vs = im.comp_vs[0];
  const int cb = chroma_at(planes + im.plane_off[1], im.plane_w[1], im.comp_w[1], im.comp_h[1], hs, vs, x, y) - 128;
  const int cr = chroma_at(planes + im.plane_off[2], im.plane_w[2], im.comp_w[2], im.comp_h[2], hs, vs, x, y) - 128;
  o[0] = clamp255(Y + ((91881 * cr + 32768) >> 16));
  o[1] = clamp255(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
  o[2] = clamp255(Y + ((116130 * cb + 32768) >> 16));
}

__global__ void jpeg_color_kernel(Batch b) {
  const ImgDev& im = b.img[blockIdx.y];
  const long long npx = (long long)im.width * im.height;
  uint8_t* out = b.out + im.out_off;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / im.width), x = (int)(i - (long long)y * im.width);
    color_pixel(im, b.planes, x, y, out + i * 3);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// progressive scans (jdphuff.c), into the same natural-order [blocks][64] buffer in frame MCU order

enum ScanKind { kDcFirst = 0, kDcRefine = 1, kAcFirst = 2, kAcRefine = 3 };

struct ScanDev {
  int img;                          // ImgDev index
  int ncomp;                        // components in the scan; 1 = non-interleaved (one block per MCU)
  int ss, se, al;
  int bpm;                          // blocks per scan MCU
  int mcus_x;                       // scan MCUs per row (the component's width in blocks when non-interleaved)
  int hs, vs, comp_first;           // non-interleaved: the component's sampling and first block in the frame MCU
  int8_t blk_slot[6];               // interleaved: scan component (table, DC predictor) of every block of the MCU
  int8_t blk_off[6];                // interleaved: the block's index within the frame MCU
};

struct ProgIvDev {
  uint64_t byte_base;               // first byte in the entropy arena
  uint32_t nbits;
  int scan;                         // ScanDev index; its Huffman tables are tabs[3 * scan + slot]
  int first_mcu, n_mcus;
};

struct ProgBatch {
  const ImgDev* img;
  const ScanDev* scan;
  const ProgIvDev* iv;
  const HuffTab* tabs;
  const uint8_t* bytes;
  int16_t* coef;
  int* err;
  const int* err_slot;
};

// frame block (MCU order, the layout jpeg_idct_kernel reads) of block k of scan MCU m
__device__ inline uint64_t frame_block(const ImgDev& im, const ScanDev& sc, int m, int k) {
  if (sc.ncomp > 1) return (uint64_t)m * im.bpm + sc.blk_off[k];
  const int by = m / sc.mcus_x, bx = m - by * sc.mcus_x;
  return (uint64_t)((by / sc.vs) * im.mcus_x + bx / sc.hs) * im.bpm + sc.comp_first + (by % sc.vs) * sc.hs + bx % sc.hs;
}

__device__ inline void prog_error(const ProgBatch& b, const ScanDev& sc, int code) {
  atomicOr(b.err + b.err_slot[sc.img], code);
}

// The sequential scan kernels give every interval a warp of its own and decode it on lane 0: intervals of different
// images or scans follow different paths, and one warp each keeps them from serialising each other.
//
// Error codes (the image's error word): 1 an invalid Huffman code, 2 an interval that ends before its last block, 4
// an EOBRUN that runs past the end of its interval.  Every read starts below the interval's last bit, so it fetches at
// most 4 bytes past it, inside the 8 zero bytes that follow every interval.

// DC first (decode_mcu_DC_first): one thread per interval, the DC difference prefix-summed per scan component from the
// interval's start, stored as (JCOEF)(sum << Al).
__device__ int dc_first(const ProgBatch& b, const ProgIvDev& iv) {
  const ScanDev& sc = b.scan[iv.scan];
  const ImgDev& im = b.img[sc.img];
  const HuffTab* tabs = b.tabs + 3 * iv.scan;
  const uint8_t* d = b.bytes + iv.byte_base;
  int16_t* coef = b.coef + im.coef_block * 64;
  int last[3] = {0, 0, 0};
  uint32_t pos = 0;
  for (int m = iv.first_mcu; m < iv.first_mcu + iv.n_mcus; ++m)
    for (int k = 0; k < sc.bpm; ++k) {
      if (pos >= iv.nbits) return 2;
      const uint32_t bits = peek32(d, pos);
      const int slot = sc.ncomp > 1 ? sc.blk_slot[k] : 0;
      int len;
      const int s = huff_decode(tabs[slot], bits, &len);
      if (s < 0) return 1;
      last[slot] += s ? extend((bits << len) >> (32 - s), s) : 0;
      pos += len + s;
      coef[frame_block(im, sc, m, k) * 64] = (int16_t)((uint32_t)last[slot] << sc.al);
    }
  return 0;
}

__global__ void jpeg_prog_dc_first_kernel(ProgBatch b, int i0, int i1) {
  const int i = i0 + (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (i >= i1 || (threadIdx.x & 31)) return;
  const ProgIvDev iv = b.iv[i];
  if (const int e = dc_first(b, iv)) prog_error(b, b.scan[iv.scan], e);
}

// DC refinement (decode_mcu_DC_refine): block t of an interval is its bit t, OR-ed in as 1 << Al.  One CUDA block per
// interval, fully parallel.
__global__ void jpeg_prog_dc_refine_kernel(ProgBatch b, int i0) {
  const ProgIvDev iv = b.iv[i0 + blockIdx.x];
  const ScanDev& sc = b.scan[iv.scan];
  const ImgDev& im = b.img[sc.img];
  const uint8_t* d = b.bytes + iv.byte_base;
  int16_t* coef = b.coef + im.coef_block * 64;
  const long long nb = (long long)iv.n_mcus * sc.bpm;
  if (threadIdx.x == 0 && nb > (long long)iv.nbits) prog_error(b, sc, 2);
  const int p1 = 1 << sc.al;
  for (long long t = threadIdx.x; t < nb && t < (long long)iv.nbits; t += blockDim.x) {
    if (!((d[t >> 3] >> (7 - (t & 7))) & 1)) continue;
    const int m = iv.first_mcu + (int)(t / sc.bpm), k = (int)(t % sc.bpm);
    int16_t& c = coef[frame_block(im, sc, m, k) * 64];
    c = (int16_t)(c | p1);
  }
}

// AC first (decode_mcu_AC_first): one thread per interval, single component, EOBRUN carried across blocks and reset
// at the interval's start.
__device__ int ac_first(const ProgBatch& b, const ProgIvDev& iv) {
  const ScanDev& sc = b.scan[iv.scan];
  const ImgDev& im = b.img[sc.img];
  const HuffTab& tab = b.tabs[3 * iv.scan];
  const uint8_t* d = b.bytes + iv.byte_base;
  int16_t* coef = b.coef + im.coef_block * 64;
  uint32_t pos = 0;
  int eobrun = 0;
  for (int m = iv.first_mcu; m < iv.first_mcu + iv.n_mcus; ++m) {
    if (eobrun > 0) {
      --eobrun;
      continue;
    }
    int16_t* blk = coef + frame_block(im, sc, m, 0) * 64;
    for (int k = sc.ss; k <= sc.se; ++k) {
      if (pos >= iv.nbits) return 2;
      const uint32_t bits = peek32(d, pos);
      int len;
      const int rs = huff_decode(tab, bits, &len);
      if (rs < 0) return 1;
      const int r = rs >> 4, s = rs & 15;
      if (s) {
        k += r;
        blk[c_natural[k < 63 ? k : 63]] = (int16_t)((uint32_t)extend((bits << len) >> (32 - s), s) << sc.al);
        pos += len + s;
      } else if (r == 15) {
        k += 15;
        pos += len;
      } else {
        eobrun = (1 << r) + (r ? (int)((bits << len) >> (32 - r)) : 0) - 1;
        pos += len + r;
        break;
      }
    }
  }
  return eobrun > 0 ? 4 : 0;
}

__global__ void jpeg_prog_ac_first_kernel(ProgBatch b, int i0, int i1) {
  const int i = i0 + (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (i >= i1 || (threadIdx.x & 31)) return;
  const ProgIvDev iv = b.iv[i];
  if (const int e = ac_first(b, iv)) prog_error(b, b.scan[iv.scan], e);
}

// AC refinement (decode_mcu_AC_refine): how many bits a block takes depends on which of its coefficients are already
// nonzero, so each interval is decoded sequentially by one thread.  A 64-bit zig-zag mask of the block's nonzero
// coefficients replaces libjpeg's coefficient-by-coefficient walk: the r zeros a symbol skips and the correction bits
// of the nonzero coefficients passed on the way are found with bit operations, and only those coefficients are read.
__device__ int ac_refine(const ProgBatch& b, const ProgIvDev& iv) {
  const ScanDev& sc = b.scan[iv.scan];
  const ImgDev& im = b.img[sc.img];
  const HuffTab& tab = b.tabs[3 * iv.scan];
  const uint8_t* d = b.bytes + iv.byte_base;
  int16_t* coef = b.coef + im.coef_block * 64;
  const int p1 = 1 << sc.al, m1 = -p1;
  const uint64_t band = (sc.se == 63 ? ~0ull : (1ull << (sc.se + 1)) - 1) & (~0ull << sc.ss);
  uint32_t pos = 0;
  int eobrun = 0;
  alignas(16) int16_t blk[64];
  // one correction bit, in stream order, for every (nonzero) coefficient of `sel`; false when the interval runs out
  auto correct = [&](uint64_t sel) {
    if ((uint64_t)pos + __popcll(sel) > iv.nbits) return false;
    uint32_t word = 0;
    int avail = 0;
    for (; sel; sel &= sel - 1) {
      if (avail == 0) {
        word = peek32(d, pos);
        avail = 32;
      }
      if (word >> 31) {
        int16_t& c = blk[c_natural[__ffsll(sel) - 1]];
        if ((c & p1) == 0) c = (int16_t)(c + (c >= 0 ? p1 : m1));
      }
      word <<= 1;
      --avail;
      ++pos;
    }
    return true;
  };
  for (int m = iv.first_mcu; m < iv.first_mcu + iv.n_mcus; ++m) {
    int4* g = reinterpret_cast<int4*>(coef + frame_block(im, sc, m, 0) * 64);
    uint64_t nat = 0;                                // nonzero coefficients, natural order
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int4 v = g[q];
      reinterpret_cast<int4*>(blk)[q] = v;
      const uint32_t w[4] = {(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        nat |= (uint64_t)((w[j] & 0xFFFFu) != 0) << (8 * q + 2 * j) | (uint64_t)((w[j] >> 16) != 0) << (8 * q + 2 * j + 1);
    }
    uint64_t nz = 0;                                 // the same in zig-zag order
#pragma unroll
    for (int k = 0; k < 64; ++k) nz |= ((nat >> c_natural[k]) & 1ull) << k;
    int k = sc.ss;
    if (eobrun == 0) {
      for (; k <= sc.se; ++k) {
        if (pos >= iv.nbits) return 2;
        const uint32_t bits = peek32(d, pos);
        int len;
        const int rs = huff_decode(tab, bits, &len);
        if (rs < 0 || (rs & 15) > 1) return 1;     // a new coefficient always has size 1
        const int r = rs >> 4;
        int s = 0;
        pos += len;
        if (rs & 15) {
          if (pos >= iv.nbits) return 2;
          s = (bits << len) >> 31 ? p1 : m1;
          ++pos;
        } else if (r != 15) {
          eobrun = (1 << r) + (r ? (int)((bits << len) >> (32 - r)) : 0);
          pos += r;
          break;
        }
        // skip r still-zero coefficients of the band, stop on the next one (or run off the band's end), and
        // append a correction bit to every nonzero coefficient passed
        const uint64_t from = band & (~0ull << k);
        uint64_t zeros = ~nz & from;
        for (int i = 0; i < r && zeros; ++i) zeros &= zeros - 1;
        const int t = zeros ? __ffsll(zeros) - 1 : sc.se + 1;
        if (!correct(nz & from & (t < 64 ? (1ull << t) - 1 : ~0ull))) return 2;
        k = t;
        if (s) {
          blk[c_natural[k < 63 ? k : 63]] = (int16_t)s;
          if (k < 64) nz |= 1ull << k;
        }
      }
    }
    if (eobrun > 0) {                                // the rest of the band of a block inside an EOB run
      if (k <= sc.se && !correct(nz & band & (~0ull << k))) return 2;
      --eobrun;
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) g[q] = reinterpret_cast<int4*>(blk)[q];
  }
  return eobrun > 0 ? 4 : 0;
}

__global__ void jpeg_prog_ac_refine_kernel(ProgBatch b, int i0, int i1) {
  const int i = i0 + (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (i >= i1 || (threadIdx.x & 31)) return;
  const ProgIvDev iv = b.iv[i];
  if (const int e = ac_refine(b, iv)) prog_error(b, b.scan[iv.scan], e);
}

// ---------------------------------------------------------------------------------------------------------------
// host parser

// one scan of a progressive file, as the decoder needs it after the whole file has been read
struct ScanInfo {
  int ncomp = 0;
  int comp[3] = {0, 0, 0};           // frame component indices, in frame order
  int ss = 0, se = 0, ah = 0, al = 0;
  int restart = 0;                   // DRI in force for this scan
  int mcus = 0;                      // MCUs of the scan (blocks of the component for a single-component scan)
  int first_iv = 0, n_iv = 0;        // its intervals in iv_start
  HuffTab tab[3];                    // per scan component: DC table (DC first) or AC table (AC scans)
};

struct Parsed {
  ibl_jpeg_info info;
  int ncomp = 0;
  int comp_id[3] = {0, 0, 0}, hs[3] = {1, 1, 1}, vs[3] = {1, 1, 1}, tq[3] = {0, 0, 0}, td[3] = {0, 0, 0},
      ta[3] = {0, 0, 0};
  uint16_t qt[4][64];
  bool qt_def[4] = {false, false, false, false};
  HuffTab dc[4], ac[4];
  bool dc_def[4] = {false, false, false, false}, ac_def[4] = {false, false, false, false};
  int restart = 0;
  int mcus_x = 0, mcus_y = 0;
  std::vector<uint8_t> entropy;      // destuffed, intervals back to back (all scans, in file order)
  std::vector<uint64_t> iv_start;    // first byte of every interval; entropy.size() closes the last
  // progressive only
  std::vector<ScanInfo> scans;
  uint16_t comp_q[3][64];            // quantisation table latched at the component's first scan (jdinput.c)
  bool comp_q_set[3] = {false, false, false};
  int coef_bits[3][64];              // libjpeg's coef_bits: -1 never coded, else the Al of the last scan coding it
  int width_blocks[3] = {0, 0, 0}, height_blocks[3] = {0, 0, 0};   // compptr->width_in_blocks / height_in_blocks
};

int reject(Parsed& p, const char* why) {
  snprintf(p.info.reason, sizeof(p.info.reason), "%s", why);
  return IBL_ERR_UNSUPPORTED;
}

// jdhuff.c jpeg_make_d_derived_tbl, with its checks; false for a table libjpeg refuses
bool build_huff(const uint8_t* counts, const uint8_t* vals, int nvals, bool is_dc, HuffTab& t) {
  memset(&t, 0, sizeof(t));
  int huffsize[257], huffcode[257];
  int p = 0;
  for (int l = 1; l <= 16; ++l) {
    const int n = counts[l - 1];
    if (p + n > 256) return false;
    for (int i = 0; i < n; ++i) huffsize[p++] = l;
  }
  huffsize[p] = 0;
  const int numsymbols = p;
  if (numsymbols != nvals) return false;
  int code = 0, si = huffsize[0];
  p = 0;
  while (huffsize[p]) {
    while (huffsize[p] == si) {
      huffcode[p++] = code;
      code++;
    }
    if (code >= (1 << si)) return false;
    code <<= 1;
    si++;
  }
  p = 0;
  for (int l = 1; l <= 16; ++l) {
    if (counts[l - 1]) {
      t.valoff[l] = p - huffcode[p];
      p += counts[l - 1];
      t.maxcode[l] = huffcode[p - 1];
    } else {
      t.maxcode[l] = -1;
    }
  }
  t.maxcode[17] = 0x7FFFFFFF;
  memcpy(t.huffval, vals, (size_t)nvals);
  p = 0;
  for (int l = 1; l <= kLookBits; ++l) {
    for (int i = 1; i <= counts[l - 1]; ++i, ++p) {
      int look = huffcode[p] << (kLookBits - l);
      for (int c = 1 << (kLookBits - l); c > 0; --c) t.look[look++] = (uint16_t)((l << 8) | vals[p]);
    }
  }
  if (is_dc)
    for (int i = 0; i < nvals; ++i)
      if (vals[i] > 15) return false;
  return true;
}

// Entropy-coded data of one scan starting at d[j]: destuff, split at RSTn (numbered from 0 in every scan), stop at
// the next other marker.  Appends the scan's intervals to p.entropy / p.iv_start and leaves j on that marker.
int read_entropy(const uint8_t* d, size_t n, size_t& j, Parsed& p) {
  const size_t first_iv = p.iv_start.size();
  p.iv_start.push_back(p.entropy.size());
  for (;;) {
    if (j >= n) return reject(p, "truncated or missing EOI marker: file ends inside the entropy-coded data");
    const uint8_t c = d[j];
    if (c != 0xFF) {
      p.entropy.push_back(c);
      ++j;
      continue;
    }
    if (j + 1 >= n) return reject(p, "truncated or missing EOI marker: file ends inside the entropy-coded data");
    const uint8_t c2 = d[j + 1];
    if (c2 == 0x00) {
      p.entropy.push_back(0xFF);
      j += 2;
    } else if (c2 == 0xFF) {
      ++j;                                        // fill byte before a marker
    } else if (c2 >= 0xD0 && c2 <= 0xD7) {
      if (c2 - 0xD0 != (int)((p.iv_start.size() - 1 - first_iv) & 7))
        return reject(p, "restart marker out of sequence");
      p.iv_start.push_back(p.entropy.size());
      j += 2;
    } else {
      return IBL_OK;
    }
  }
}

// Progressive scan header after the component list (jdphuff.c start_pass_phuff_decoder): its range checks, which
// libjpeg errors on, and the coef_bits bookkeeping whose JWRN_BOGUS_PROGRESSION warnings are rejected here too.
int progressive_scan(Parsed& p, ScanInfo& sc, const uint8_t* ssz) {
  sc.ss = ssz[0];
  sc.se = ssz[1];
  sc.ah = ssz[2] >> 4;
  sc.al = ssz[2] & 15;
  if (sc.ss == 0) {
    if (sc.se != 0) return reject(p, "bad progression: DC scan with Se != 0");
  } else {
    if (sc.ss > sc.se || sc.se > 63) return reject(p, "bad progression: spectral band out of range");
    if (sc.ncomp != 1) return reject(p, "bad progression: AC scan with more than one component");
  }
  if (sc.ah != 0 && sc.al != sc.ah - 1) return reject(p, "bad progression: refinement with Al != Ah - 1");
  if (sc.al > 13) return reject(p, "bad progression: Al > 13");
  for (int i = 0; i < sc.ncomp; ++i) {
    int* cb = p.coef_bits[sc.comp[i]];
    if (sc.ss > 0 && cb[0] < 0) return reject(p, "bogus progression: AC scan before the component's DC scan");
    for (int k = sc.ss; k <= sc.se; ++k) {
      if (sc.ah != (cb[k] < 0 ? 0 : cb[k])) return reject(p, "bogus progression: Ah differs from the previous Al");
      cb[k] = sc.al;
    }
  }
  for (int i = 0; i < sc.ncomp; ++i) {
    const int c = sc.comp[i];
    if (sc.ss == 0 && sc.ah == 0) {
      if (!p.dc_def[p.td[c]]) return reject(p, "missing Huffman table");
      sc.tab[i] = p.dc[p.td[c]];                     // snapshot: DHT may redefine it before a later scan
    } else if (sc.ss > 0) {
      if (!p.ac_def[p.ta[c]]) return reject(p, "missing Huffman table");
      sc.tab[i] = p.ac[p.ta[c]];
    }
    if (!p.comp_q_set[c]) {                          // jdinput.c latch_quant_tables
      if (!p.qt_def[p.tq[c]]) return reject(p, "missing quantisation table");
      memcpy(p.comp_q[c], p.qt[p.tq[c]], sizeof(p.comp_q[c]));
      p.comp_q_set[c] = true;
    }
  }
  return IBL_OK;
}

// Baseline (SOF0/SOF1, one interleaved scan) or, with `progressive`, progressive Huffman (SOF2, any valid scan
// script).  Both share the marker reader, the Huffman table derivation, the component and sampling rules and the
// destuffing; each rejects the other kind.
int parse_jpeg(const uint8_t* d, size_t n, Parsed& p, bool progressive = false) {
  memset(&p.info, 0, sizeof(p.info));
  if (!d || n < 4 || d[0] != 0xFF || d[1] != 0xD8) return reject(p, "not a JPEG file (no SOI marker)");
  size_t i = 2;
  bool sof = false, sos = false, jfif = false, adobe = false;
  int adobe_transform = -1, width = 0, height = 0;
  if (progressive)
    for (int c = 0; c < 3; ++c)
      for (int k = 0; k < 64; ++k) p.coef_bits[c][k] = -1;
  for (;;) {
    if (i >= n) return reject(p, sos ? "missing EOI marker" : "truncated: file ends before the scan");
    if (d[i] != 0xFF) return reject(p, "extraneous bytes between segments");
    while (i < n && d[i] == 0xFF) ++i;
    if (i >= n) return reject(p, sos ? "missing EOI marker" : "truncated: file ends before the scan");
    const int m = d[i++];
    if (m == 0xD9) {
      if (!sos) return reject(p, "EOI before any scan");
      break;
    }
    if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01 || m == 0x00) return reject(p, "unexpected marker");
    if (i + 2 > n) return reject(p, "truncated: segment header cut short");
    const size_t L = ((size_t)d[i] << 8) | d[i + 1];
    if (L < 2) return reject(p, "bad segment length");
    if (i + L > n) return reject(p, "truncated: segment runs past the end of the file");
    const uint8_t* seg = d + i + 2;
    const size_t sl = L - 2;
    i += L;
    if (sos && m != 0xDA && !(m >= 0xE0 && m <= 0xEF) && m != 0xFE && m != 0xC4 && m != 0xDB && m != 0xDD)
      return reject(p, "unsupported marker after the scan");
    switch (m) {
      case 0xC0:
      case 0xC1:
      case 0xC2: {
        if (m == 0xC2 && !progressive) return reject(p, "progressive");
        if (m != 0xC2 && progressive) return reject(p, "sequential (not progressive)");
        if (sof) return reject(p, "more than one frame");
        if (sl < 6) return reject(p, "bad segment length");
        if (seg[0] != 8) return reject(p, "12-bit (not 8-bit) samples");
        height = (seg[1] << 8) | seg[2];
        width = (seg[3] << 8) | seg[4];
        const int nf = seg[5];
        if (sl != 6 + 3 * (size_t)nf) return reject(p, "bad segment length");
        if (height == 0) return reject(p, "height defined by a DNL marker");
        if (width == 0) return reject(p, "zero width");
        if (nf == 4) return reject(p, "4 components (CMYK/YCCK)");
        if (nf != 1 && nf != 3) return reject(p, "component count other than 1 or 3");
        p.ncomp = nf;
        for (int c = 0; c < nf; ++c) {
          p.comp_id[c] = seg[6 + 3 * c];
          p.hs[c] = seg[7 + 3 * c] >> 4;
          p.vs[c] = seg[7 + 3 * c] & 15;
          p.tq[c] = seg[8 + 3 * c];
          if (p.hs[c] < 1 || p.hs[c] > 4 || p.vs[c] < 1 || p.vs[c] > 4 || p.tq[c] > 3)
            return reject(p, "bad frame component");
        }
        sof = true;
        break;
      }
      case 0xC6: return reject(p, "progressive");
      case 0xC3: case 0xC7: return reject(p, "lossless");
      case 0xC5: case 0xDE: case 0xDF: return reject(p, "hierarchical");
      case 0xC9: case 0xCA: case 0xCB: case 0xCD: case 0xCE: case 0xCF: case 0xCC:
        return reject(p, "arithmetic coding");
      case 0xC4: {
        size_t k = 0;
        while (k < sl) {
          if (k + 17 > sl) return reject(p, "bad segment length");
          const int tc = seg[k] >> 4, th = seg[k] & 15;
          if (tc > 1 || th > 3) return reject(p, "bad Huffman table");
          int total = 0;
          for (int l = 0; l < 16; ++l) total += seg[k + 1 + l];
          if (total > 256 || k + 17 + total > sl) return reject(p, "bad segment length");
          if (!build_huff(seg + k + 1, seg + k + 17, total, tc == 0, tc == 0 ? p.dc[th] : p.ac[th]))
            return reject(p, "bad Huffman table");
          (tc == 0 ? p.dc_def : p.ac_def)[th] = true;
          k += 17 + total;
        }
        break;
      }
      case 0xDB: {
        size_t k = 0;
        while (k < sl) {
          const int pq = seg[k] >> 4, tq = seg[k] & 15;
          if (pq > 1 || tq > 3) return reject(p, "bad quantisation table");
          if (k + 1 + 64 * (pq + 1) > sl) return reject(p, "bad segment length");
          for (int z = 0; z < 64; ++z)
            p.qt[tq][h_natural[z]] = pq ? (uint16_t)((seg[k + 1 + 2 * z] << 8) | seg[k + 2 + 2 * z]) : seg[k + 1 + z];
          p.qt_def[tq] = true;
          k += 1 + 64 * (pq + 1);
        }
        break;
      }
      case 0xDD:
        if (sl != 2) return reject(p, "bad segment length");
        p.restart = (seg[0] << 8) | seg[1];
        break;
      case 0xDA: {
        if (!sof) return reject(p, "scan before the frame header");
        if (sos && !progressive) return reject(p, "multi-scan");
        if (sl < 1) return reject(p, "bad segment length");
        const int ns = seg[0];
        if (sl != 4 + 2 * (size_t)ns) return reject(p, "bad segment length");
        ScanInfo sc;
        if (!progressive) {
          if (ns != p.ncomp) return reject(p, "multi-scan (components in separate scans)");
          for (int c = 0; c < ns; ++c) {
            if (seg[1 + 2 * c] != p.comp_id[c]) return reject(p, "scan component order differs from the frame");
            p.td[c] = seg[2 + 2 * c] >> 4;
            p.ta[c] = seg[2 + 2 * c] & 15;
            if (p.td[c] > 3 || p.ta[c] > 3) return reject(p, "bad scan header");
          }
          const uint8_t* ssz = seg + 1 + 2 * ns;
          if (ssz[0] != 0 || ssz[1] != 63 || ssz[2] != 0) return reject(p, "not a sequential scan");
          for (int c = 0; c < ns; ++c) {
            if (!p.qt_def[p.tq[c]]) return reject(p, "missing quantisation table");
            if (!p.dc_def[p.td[c]] || !p.ac_def[p.ta[c]]) return reject(p, "missing Huffman table");
          }
        } else {
          if (ns < 1 || ns > p.ncomp) return reject(p, "bad scan header");
          sc.ncomp = ns;
          for (int s = 0, c = 0; s < ns; ++s, ++c) {
            while (c < p.ncomp && p.comp_id[c] != seg[1 + 2 * s]) ++c;
            if (c == p.ncomp) return reject(p, "scan component order differs from the frame");
            sc.comp[s] = c;
            p.td[c] = seg[2 + 2 * s] >> 4;
            p.ta[c] = seg[2 + 2 * s] & 15;
            if (p.td[c] > 3 || p.ta[c] > 3) return reject(p, "bad scan header");
          }
        }
        // colour space as libjpeg decides it (jdapimin.c default_decompress_parms)
        if (!sos && p.ncomp == 3) {
          bool rgb = false;
          if (jfif) rgb = false;
          else if (adobe) rgb = adobe_transform == 0;
          else rgb = p.comp_id[0] == 'R' && p.comp_id[1] == 'G' && p.comp_id[2] == 'B';
          if (rgb) return reject(p, "RGB-coded (no YCbCr transform)");
          const bool chroma11 = p.hs[1] == 1 && p.vs[1] == 1 && p.hs[2] == 1 && p.vs[2] == 1;
          const bool luma_ok = (p.hs[0] == 1 && p.vs[0] == 1) || (p.hs[0] == 2 && p.vs[0] == 1) ||
                               (p.hs[0] == 2 && p.vs[0] == 2);
          if (!chroma11 || !luma_ok) return reject(p, "sampling other than 4:4:4, 4:2:2 or 4:2:0");
          p.mcus_x = (width + 8 * p.hs[0] - 1) / (8 * p.hs[0]);
          p.mcus_y = (height + 8 * p.vs[0] - 1) / (8 * p.vs[0]);
        } else if (!sos) {
          p.hs[0] = p.vs[0] = 1;                       // one component: one block per MCU whatever its factors
          p.mcus_x = (width + 7) / 8;
          p.mcus_y = (height + 7) / 8;
        }
        long long mcus = (long long)p.mcus_x * p.mcus_y;
        if (progressive) {
          if (!sos)
            for (int c = 0; c < p.ncomp; ++c) {        // jdinput.c initial_setup: ceil(size * samp / (max_samp * 8))
              p.width_blocks[c] = (int)(((long long)width * p.hs[c] + 8 * p.hs[0] - 1) / (8 * p.hs[0]));
              p.height_blocks[c] = (int)(((long long)height * p.vs[c] + 8 * p.vs[0] - 1) / (8 * p.vs[0]));
            }
          IBL_RET(progressive_scan(p, sc, seg + 1 + 2 * ns));
          if (ns == 1) mcus = (long long)p.width_blocks[sc.comp[0]] * p.height_blocks[sc.comp[0]];
          sc.restart = p.restart;
          sc.mcus = (int)mcus;
          sc.first_iv = (int)p.iv_start.size();
        } else {
          p.entropy.clear();
          p.iv_start.clear();
        }
        if (!sos) p.entropy.reserve(n - i);
        size_t j = i;
        IBL_RET(read_entropy(d, n, j, p));
        i = j;
        const long long n_iv = (long long)p.iv_start.size() - sc.first_iv;
        const long long want = p.restart ? (mcus + p.restart - 1) / p.restart : 1;
        if (n_iv != want) return reject(p, "restart markers do not match the restart interval");
        if (progressive) {
          sc.n_iv = (int)n_iv;
          p.scans.push_back(sc);
        }
        sos = true;
        break;
      }
      case 0xE0:
        if (sl >= 5 && memcmp(seg, "JFIF\0", 5) == 0) jfif = true;
        break;
      case 0xEE:
        if (sl >= 12 && memcmp(seg, "Adobe", 5) == 0) {
          adobe = true;
          adobe_transform = seg[11];
        }
        break;
      case 0xDC: return reject(p, "height defined by a DNL marker");
      default:
        if ((m >= 0xE0 && m <= 0xEF) || m == 0xFE) break;   // APPn, COM
        return reject(p, "unsupported marker");
    }
  }
  // libjpeg reads frame and scan before it decides: JFIF/Adobe may come after SOF, so the check above runs at SOS
  p.info.width = width;
  p.info.height = height;
  p.info.components = p.ncomp;
  p.info.h_samp = p.hs[0];
  p.info.v_samp = p.vs[0];
  p.info.restart_interval = p.restart;
  p.info.intervals = (int)p.iv_start.size();
  p.info.mcus = p.mcus_x * p.mcus_y;
  p.info.entropy_bytes = p.entropy.size();
  // jdcoefct.c smoothing_ok: libjpeg smooths the blocks of a progressive file when the DC or one of the first nine
  // AC coefficients (SAVED_COEFS) of a component is not fully refined after the last scan; such files stay on the host
  if (progressive)
    for (int c = 0; c < p.ncomp; ++c)
      for (int k = 0; k < 10; ++k)
        if (p.coef_bits[c][k] != 0) return reject(p, "block smoothing (a low-frequency coefficient not fully refined)");
  return IBL_OK;
}

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

}  // namespace

void jpeg_ws_destroy(JpegWs* ws) {
  if (!ws) return;
  if (ws->pending) cudaEventSynchronize(ws->copied);
  if (ws->host) cudaFreeHost(ws->host);
  if (ws->blob) cudaFree(ws->blob);
  if (ws->arena) cudaFree(ws->arena);
  if (ws->copied) cudaEventDestroy(ws->copied);
  delete ws;
}

int grow_device(void** p, size_t* cap, size_t need) {
  if (need <= *cap) return IBL_OK;
  if (*p) cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  const cudaError_t e = cudaMalloc(p, need);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_last_error("jpeg workspace cudaMalloc(" + std::to_string(need) + " B) failed: " + cudaGetErrorString(e));
    return IBL_ERR_OOM;
  }
  *cap = need;
  return IBL_OK;
}

int ws_open(JpegWs** pws) {
  if (!*pws) {
    *pws = new (std::nothrow) JpegWs();
    if (!*pws) return IBL_ERR_OOM;
    IBL_CUDA_OK(cudaEventCreateWithFlags(&(*pws)->copied, cudaEventDisableTiming));
  }
  return IBL_OK;
}

// pinned staging of at least `bytes`, once the previous call's H2D copy no longer reads it
int stage_host(JpegWs* ws, size_t bytes) {
  if (ws->pending) {
    IBL_CUDA_OK(cudaEventSynchronize(ws->copied));
    ws->pending = false;
  }
  if (ws->host_cap < bytes) {
    if (ws->host) cudaFreeHost(ws->host);
    ws->host = nullptr;
    ws->host_cap = 0;
    if (cudaMallocHost(&ws->host, bytes) != cudaSuccess) {
      cudaGetLastError();
      set_last_error("jpeg staging cudaMallocHost failed");
      return IBL_ERR_OOM;
    }
    ws->host_cap = bytes;
  }
  return IBL_OK;
}

// frame layout of one parsed image: MCU grid, blocks per MCU, component planes at libjpeg's sizes, quantisation
// tables q[c]; reserves its coefficient blocks and plane bytes
static void fill_img(const Parsed& p, const uint16_t (*q)[64], ImgDev& im, uint64_t& coef_blocks,
                     uint64_t& plane_bytes) {
  memset(&im, 0, sizeof(im));
  im.width = p.info.width;
  im.height = p.info.height;
  im.ncomp = p.ncomp;
  im.mcus_x = p.mcus_x;
  im.mcus_y = p.mcus_y;
  const int hmax = p.hs[0], vmax = p.vs[0];
  int k = 0;
  for (int c = 0; c < p.ncomp; ++c) {
    im.comp_hs[c] = p.hs[c];
    im.comp_vs[c] = p.vs[c];
    for (int v = 0; v < p.vs[c]; ++v)
      for (int h = 0; h < p.hs[c]; ++h, ++k) {
        im.blk_comp[k] = (int8_t)c;
        im.blk_dx[k] = (int8_t)h;
        im.blk_dy[k] = (int8_t)v;
      }
    im.comp_w[c] = (int)(((long long)im.width * p.hs[c] + hmax - 1) / hmax);
    im.comp_h[c] = (int)(((long long)im.height * p.vs[c] + vmax - 1) / vmax);
    im.plane_w[c] = im.mcus_x * p.hs[c] * 8;
    im.plane_off[c] = plane_bytes;
    plane_bytes += align16((uint64_t)im.plane_w[c] * im.mcus_y * p.vs[c] * 8);
    memcpy(im.q[c], q[c], sizeof(im.q[c]));
  }
  im.bpm = k;
  im.nblocks = im.mcus_x * im.mcus_y * im.bpm;
  im.coef_block = coef_blocks;
  coef_blocks += im.nblocks;
}

int jpeg_decode_u8(JpegWs** pws, const uint8_t* const* files, const size_t* lens, int N, uint8_t* out_u8,
                   const uint64_t* out_offsets, int* status, int* err_dev, cudaStream_t s, uint64_t* launches) {
  IBL_RET(ws_open(pws));
  JpegWs* ws = *pws;
  IBL_CUDA_OK(cudaMemsetAsync(err_dev, 0, (size_t)N * sizeof(int), s));
  std::vector<Parsed> ps;
  std::vector<int> slot;
  for (int n = 0; n < N; ++n) {
    Parsed p;
    status[n] = files[n] ? parse_jpeg(files[n], lens[n], p) : IBL_ERR_BAD_ARG;
    if (status[n] != IBL_OK) continue;
    ps.push_back(std::move(p));
    slot.push_back(n);
  }
  const int M = (int)ps.size();
  if (M == 0) return IBL_OK;
  // layout
  std::vector<ImgDev> imgs(M);
  std::vector<IntervalDev> ivs;
  std::vector<int> seq_iv;
  uint64_t ebytes = 0, coef_blocks = 0, plane_bytes = 0;
  for (int m = 0; m < M; ++m) {
    const Parsed& p = ps[m];
    ImgDev& im = imgs[m];
    uint16_t q[3][64];
    for (int c = 0; c < p.ncomp; ++c) memcpy(q[c], p.qt[p.tq[c]], sizeof(q[c]));
    fill_img(p, q, im, coef_blocks, plane_bytes);
    im.out_off = out_offsets[slot[m]];
    im.first_seq = (int)seq_iv.size();
    const int n_iv = (int)p.iv_start.size();
    const long long mcus = (long long)im.mcus_x * im.mcus_y;
    for (int t = 0; t < n_iv; ++t) {
      IntervalDev iv;
      const uint64_t b0 = p.iv_start[t], b1 = t + 1 < n_iv ? p.iv_start[t + 1] : p.entropy.size();
      if ((b1 - b0) * 8 > 0xFFFFFFFFull - 2ull * kRunBits) {
        status[slot[m]] = IBL_ERR_UNSUPPORTED;          // cannot happen below 512 MB per interval
        return IBL_ERR_UNSUPPORTED;
      }
      iv.byte_base = ebytes;
      iv.nbits = (uint32_t)((b1 - b0) * 8);
      iv.img = m;
      const long long mcu0 = p.restart ? (long long)t * p.restart : 0;
      const long long mcu1 = p.restart ? std::min(mcus, mcu0 + p.restart) : mcus;
      iv.first_block = (int)(mcu0 * im.bpm);
      iv.nblocks = (int)((mcu1 - mcu0) * im.bpm);
      iv.first_seq = (int)seq_iv.size();
      iv.n_seq = std::max(1, (int)((iv.nbits + kRunBits - 1) / kRunBits));
      for (int q = 0; q < iv.n_seq; ++q) seq_iv.push_back((int)ivs.size());
      ivs.push_back(iv);
      ebytes += (b1 - b0) + kPad;
    }
    im.n_seq = (int)seq_iv.size() - im.first_seq;
  }
  const int NS = (int)seq_iv.size(), NI = (int)ivs.size();
  // staging blob: images | intervals | Huffman tables | run -> interval | slots | entropy bytes
  const size_t o_img = 0, o_iv = align16(o_img + sizeof(ImgDev) * M), o_tab = align16(o_iv + sizeof(IntervalDev) * NI),
               o_seq = align16(o_tab + sizeof(HuffTab) * 6 * M), o_slot = align16(o_seq + sizeof(int) * NS),
               o_bytes = align16(o_slot + sizeof(int) * M), blob_bytes = align16(o_bytes + ebytes);
  IBL_RET(stage_host(ws, blob_bytes));
  uint8_t* h = ws->host;
  memcpy(h + o_img, imgs.data(), sizeof(ImgDev) * M);
  memcpy(h + o_iv, ivs.data(), sizeof(IntervalDev) * NI);
  HuffTab* tabs = reinterpret_cast<HuffTab*>(h + o_tab);
  for (int m = 0; m < M; ++m)
    for (int c = 0; c < ps[m].ncomp; ++c) {
      tabs[6 * m + 2 * c] = ps[m].dc[ps[m].td[c]];
      tabs[6 * m + 2 * c + 1] = ps[m].ac[ps[m].ta[c]];
    }
  memcpy(h + o_seq, seq_iv.data(), sizeof(int) * NS);
  memcpy(h + o_slot, slot.data(), sizeof(int) * M);
  {
    uint8_t* e = h + o_bytes;
    for (int m = 0; m < M; ++m) {
      const Parsed& p = ps[m];
      const int n_iv = (int)p.iv_start.size();
      for (int t = 0; t < n_iv; ++t) {
        const uint64_t b0 = p.iv_start[t], b1 = t + 1 < n_iv ? p.iv_start[t + 1] : p.entropy.size();
        memcpy(e, p.entropy.data() + b0, b1 - b0);
        memset(e + (b1 - b0), 0, kPad);
        e += (b1 - b0) + kPad;
      }
    }
  }
  // device arena: states | new states | counts | new counts | first blocks | flags | coefficients | planes
  const size_t a_st = 0, a_stn = a_st + 8 * (size_t)NS, a_cnt = a_stn + 8 * (size_t)NS, a_cntn = align16(a_cnt + 4 * (size_t)NS),
               a_first = align16(a_cntn + 4 * (size_t)NS), a_need = align16(a_first + 4 * (size_t)NS),
               a_chg = align16(a_need + NS), a_coef = align16(a_chg + NS),
               a_planes = align16(a_coef + coef_blocks * 64 * sizeof(int16_t)), arena_bytes = align16(a_planes + plane_bytes);
  IBL_RET(grow_device(&ws->blob, &ws->blob_cap, blob_bytes));
  IBL_RET(grow_device(&ws->arena, &ws->arena_cap, arena_bytes));
  IBL_CUDA_OK(cudaMemcpyAsync(ws->blob, ws->host, blob_bytes, cudaMemcpyHostToDevice, s));
  IBL_CUDA_OK(cudaEventRecord(ws->copied, s));
  ws->pending = true;
  uint8_t* db = static_cast<uint8_t*>(ws->blob);
  uint8_t* da = static_cast<uint8_t*>(ws->arena);
  Batch b;
  b.img = reinterpret_cast<const ImgDev*>(db + o_img);
  b.iv = reinterpret_cast<const IntervalDev*>(db + o_iv);
  b.tabs = reinterpret_cast<const HuffTab*>(db + o_tab);
  b.seq_iv = reinterpret_cast<const int*>(db + o_seq);
  b.err_slot = reinterpret_cast<const int*>(db + o_slot);
  b.bytes = db + o_bytes;
  b.n_seq = NS;
  b.st = reinterpret_cast<uint64_t*>(da + a_st);
  b.st_new = reinterpret_cast<uint64_t*>(da + a_stn);
  b.cnt = reinterpret_cast<int*>(da + a_cnt);
  b.cnt_new = reinterpret_cast<int*>(da + a_cntn);
  b.first_blk = reinterpret_cast<int*>(da + a_first);
  b.need = da + a_need;
  b.chg = da + a_chg;
  b.coef = reinterpret_cast<int16_t*>(da + a_coef);
  b.planes = da + a_planes;
  b.out = out_u8;
  b.err = err_dev;
  IBL_CUDA_OK(cudaMemsetAsync(b.coef, 0, coef_blocks * 64 * sizeof(int16_t), s));
  const int sms = device_sm_count();
  auto grid1 = [&](long long work, int threads) {
    const long long g = (work + threads - 1) / threads;
    return (unsigned)std::max(1ll, std::min(g, (long long)sms * 16));
  };
  int max_blocks = 0;
  long long max_px = 0;
  for (const ImgDev& im : imgs) {
    max_blocks = std::max(max_blocks, im.nblocks);
    max_px = std::max(max_px, (long long)im.width * im.height);
  }
  jpeg_sync_kernel<<<grid1(NS, 128), 128, 0, s>>>(b);
  jpeg_fix_kernel<<<M, kFixThreads, 0, s>>>(b);
  jpeg_write_kernel<<<grid1(NS, 128), 128, 0, s>>>(b);
  jpeg_dc_kernel<<<NI, kDcThreads, 0, s>>>(b);
  jpeg_idct_kernel<<<dim3(std::min(grid1(max_blocks, 128), 1024u), M), 128, 0, s>>>(b);
  jpeg_color_kernel<<<dim3(std::min(grid1(max_px, 256), 1024u), M), 256, 0, s>>>(b);
  IBL_CUDA_OK(cudaGetLastError());
  if (launches) *launches += 6;
  return IBL_OK;
}

// Progressive files: the parser records the scan script; the scans of one image run in file order, one launch per
// (scan round, scan kind) covering that scan of every image of the batch, then the baseline IDCT and colour kernels.
int jpeg_decode_progressive_u8(JpegWs** pws, const uint8_t* const* files, const size_t* lens, int N, uint8_t* out_u8,
                               const uint64_t* out_offsets, int* status, int* err_dev, cudaStream_t s,
                               uint64_t* launches) {
  IBL_RET(ws_open(pws));
  JpegWs* ws = *pws;
  IBL_CUDA_OK(cudaMemsetAsync(err_dev, 0, (size_t)N * sizeof(int), s));
  std::vector<Parsed> ps;
  std::vector<int> slot;
  for (int n = 0; n < N; ++n) {
    Parsed p;
    status[n] = files[n] ? parse_jpeg(files[n], lens[n], p, true) : IBL_ERR_BAD_ARG;
    if (status[n] != IBL_OK) continue;
    ps.push_back(std::move(p));
    slot.push_back(n);
  }
  const int M = (int)ps.size();
  if (M == 0) return IBL_OK;
  // layout: frames, scans (in image order), entropy bytes per image in file order
  std::vector<ImgDev> imgs(M);
  std::vector<ScanDev> scans;
  std::vector<int> scan0(M);                         // first ScanDev of every image
  std::vector<std::vector<uint64_t>> iv_base(M);     // arena byte of every interval of every image
  uint64_t ebytes = 0, coef_blocks = 0, plane_bytes = 0;
  int rounds = 0;
  for (int m = 0; m < M; ++m) {
    const Parsed& p = ps[m];
    fill_img(p, p.comp_q, imgs[m], coef_blocks, plane_bytes);
    imgs[m].out_off = out_offsets[slot[m]];
    int comp_first[3] = {0, 0, 0};
    for (int c = 1; c < p.ncomp; ++c) comp_first[c] = comp_first[c - 1] + p.hs[c - 1] * p.vs[c - 1];
    scan0[m] = (int)scans.size();
    rounds = std::max(rounds, (int)p.scans.size());
    for (const ScanInfo& si : p.scans) {
      ScanDev sd;
      memset(&sd, 0, sizeof(sd));
      sd.img = m;
      sd.ncomp = si.ncomp;
      sd.ss = si.ss;
      sd.se = si.se;
      sd.al = si.al;
      if (si.ncomp > 1) {
        sd.mcus_x = p.mcus_x;
        for (int i = 0; i < si.ncomp; ++i) {
          const int c = si.comp[i];
          for (int v = 0; v < p.vs[c]; ++v)
            for (int h = 0; h < p.hs[c]; ++h, ++sd.bpm) {
              sd.blk_slot[sd.bpm] = (int8_t)i;
              sd.blk_off[sd.bpm] = (int8_t)(comp_first[c] + v * p.hs[c] + h);
            }
        }
      } else {
        const int c = si.comp[0];
        sd.bpm = 1;
        sd.mcus_x = p.width_blocks[c];
        sd.hs = p.hs[c];
        sd.vs = p.vs[c];
        sd.comp_first = comp_first[c];
      }
      scans.push_back(sd);
    }
    const size_t n_iv = p.iv_start.size();
    for (size_t t = 0; t < n_iv; ++t) {
      const uint64_t b0 = p.iv_start[t], b1 = t + 1 < n_iv ? p.iv_start[t + 1] : p.entropy.size();
      if ((b1 - b0) * 8 > 0xFFFFFFFFull - 64) {
        status[slot[m]] = IBL_ERR_UNSUPPORTED;       // cannot happen below 512 MB per interval
        return IBL_ERR_UNSUPPORTED;
      }
      iv_base[m].push_back(ebytes);
      ebytes += (b1 - b0) + kPad;
    }
  }
  // intervals grouped by (round, kind): round r holds the r-th scan of every image
  std::vector<ProgIvDev> ivs;
  std::vector<int> group(4 * rounds + 1, 0);
  for (int r = 0; r < rounds; ++r)
    for (int kind = 0; kind < 4; ++kind) {
      group[4 * r + kind] = (int)ivs.size();
      for (int m = 0; m < M; ++m) {
        const Parsed& p = ps[m];
        if (r >= (int)p.scans.size()) continue;
        const ScanInfo& si = p.scans[r];
        if ((si.ss == 0 ? 0 : 2) + (si.ah == 0 ? 0 : 1) != kind) continue;
        for (int t = 0; t < si.n_iv; ++t) {
          const int g = si.first_iv + t;
          const uint64_t b0 = p.iv_start[g], b1 = g + 1 < (int)p.iv_start.size() ? p.iv_start[g + 1] : p.entropy.size();
          ProgIvDev iv;
          iv.byte_base = iv_base[m][g];
          iv.nbits = (uint32_t)((b1 - b0) * 8);
          iv.scan = scan0[m] + r;
          iv.first_mcu = si.restart ? t * si.restart : 0;
          iv.n_mcus = si.restart ? std::min(si.mcus - iv.first_mcu, si.restart) : si.mcus;
          ivs.push_back(iv);
        }
      }
    }
  group[4 * rounds] = (int)ivs.size();
  const int NSC = (int)scans.size(), NI = (int)ivs.size();
  // staging blob: images | scans | intervals | Huffman tables | slots | entropy bytes
  const size_t o_img = 0, o_scan = align16(o_img + sizeof(ImgDev) * M),
               o_iv = align16(o_scan + sizeof(ScanDev) * NSC), o_tab = align16(o_iv + sizeof(ProgIvDev) * NI),
               o_slot = align16(o_tab + sizeof(HuffTab) * 3 * NSC), o_bytes = align16(o_slot + sizeof(int) * M),
               blob_bytes = align16(o_bytes + ebytes);
  IBL_RET(stage_host(ws, blob_bytes));
  uint8_t* h = ws->host;
  memcpy(h + o_img, imgs.data(), sizeof(ImgDev) * M);
  memcpy(h + o_scan, scans.data(), sizeof(ScanDev) * NSC);
  memcpy(h + o_iv, ivs.data(), sizeof(ProgIvDev) * NI);
  HuffTab* tabs = reinterpret_cast<HuffTab*>(h + o_tab);
  for (int m = 0; m < M; ++m)
    for (size_t r = 0; r < ps[m].scans.size(); ++r)
      for (int i = 0; i < 3; ++i) tabs[3 * (scan0[m] + r) + i] = ps[m].scans[r].tab[i];
  memcpy(h + o_slot, slot.data(), sizeof(int) * M);
  for (int m = 0; m < M; ++m) {
    const Parsed& p = ps[m];
    const size_t n_iv = p.iv_start.size();
    for (size_t t = 0; t < n_iv; ++t) {
      const uint64_t b0 = p.iv_start[t], b1 = t + 1 < n_iv ? p.iv_start[t + 1] : p.entropy.size();
      uint8_t* e = h + o_bytes + iv_base[m][t];
      memcpy(e, p.entropy.data() + b0, b1 - b0);
      memset(e + (b1 - b0), 0, kPad);
    }
  }
  // device arena: coefficients | planes
  const size_t a_coef = 0, a_planes = align16(a_coef + coef_blocks * 64 * sizeof(int16_t)),
               arena_bytes = align16(a_planes + plane_bytes);
  IBL_RET(grow_device(&ws->blob, &ws->blob_cap, blob_bytes));
  IBL_RET(grow_device(&ws->arena, &ws->arena_cap, arena_bytes));
  IBL_CUDA_OK(cudaMemcpyAsync(ws->blob, ws->host, blob_bytes, cudaMemcpyHostToDevice, s));
  IBL_CUDA_OK(cudaEventRecord(ws->copied, s));
  ws->pending = true;
  uint8_t* db = static_cast<uint8_t*>(ws->blob);
  uint8_t* da = static_cast<uint8_t*>(ws->arena);
  ProgBatch pb;
  pb.img = reinterpret_cast<const ImgDev*>(db + o_img);
  pb.scan = reinterpret_cast<const ScanDev*>(db + o_scan);
  pb.iv = reinterpret_cast<const ProgIvDev*>(db + o_iv);
  pb.tabs = reinterpret_cast<const HuffTab*>(db + o_tab);
  pb.err_slot = reinterpret_cast<const int*>(db + o_slot);
  pb.bytes = db + o_bytes;
  pb.coef = reinterpret_cast<int16_t*>(da + a_coef);
  pb.err = err_dev;
  Batch b;
  memset(&b, 0, sizeof(b));
  b.img = pb.img;
  b.coef = pb.coef;
  b.planes = da + a_planes;
  b.out = out_u8;
  IBL_CUDA_OK(cudaMemsetAsync(pb.coef, 0, coef_blocks * 64 * sizeof(int16_t), s));
  uint64_t n_launch = 2;
  for (int r = 0; r < rounds; ++r)
    for (int kind = 0; kind < 4; ++kind) {
      const int i0 = group[4 * r + kind], i1 = group[4 * r + kind + 1];
      if (i0 == i1) continue;
      const unsigned warps = (unsigned)((i1 - i0 + kProgWarps - 1) / kProgWarps);
      switch (kind) {
        case kDcFirst: jpeg_prog_dc_first_kernel<<<warps, 32 * kProgWarps, 0, s>>>(pb, i0, i1); break;
        case kDcRefine: jpeg_prog_dc_refine_kernel<<<(unsigned)(i1 - i0), 256, 0, s>>>(pb, i0); break;
        case kAcFirst: jpeg_prog_ac_first_kernel<<<warps, 32 * kProgWarps, 0, s>>>(pb, i0, i1); break;
        default: jpeg_prog_ac_refine_kernel<<<warps, 32 * kProgWarps, 0, s>>>(pb, i0, i1); break;
      }
      ++n_launch;
    }
  const int sms = device_sm_count();
  auto grid1 = [&](long long work, int threads) {
    const long long g = (work + threads - 1) / threads;
    return (unsigned)std::max(1ll, std::min(g, (long long)sms * 16));
  };
  int max_blocks = 0;
  long long max_px = 0;
  for (const ImgDev& im : imgs) {
    max_blocks = std::max(max_blocks, im.nblocks);
    max_px = std::max(max_px, (long long)im.width * im.height);
  }
  jpeg_idct_kernel<<<dim3(std::min(grid1(max_blocks, 128), 1024u), M), 128, 0, s>>>(b);
  jpeg_color_kernel<<<dim3(std::min(grid1(max_px, 256), 1024u), M), 256, 0, s>>>(b);
  IBL_CUDA_OK(cudaGetLastError());
  if (launches) *launches += n_launch;
  return IBL_OK;
}

}  // namespace ibl

extern "C" int ibl_jpeg_parse(const uint8_t* data, size_t len, ibl_jpeg_info* out) {
  IBL_REQUIRE(out, "null argument");
  ibl::Parsed p;
  const int st = ibl::parse_jpeg(data, len, p);
  *out = p.info;
  if (st != IBL_OK) ibl::set_last_error(std::string("ibl_jpeg_parse: ") + p.info.reason);
  return st;
}

extern "C" int ibl_jpeg_parse_progressive(const uint8_t* data, size_t len, ibl_jpeg_info* out, int* n_scans,
                                          ibl_jpeg_scan* scans, int max_scans) {
  IBL_REQUIRE(out, "null argument");
  ibl::Parsed p;
  const int st = ibl::parse_jpeg(data, len, p, true);
  *out = p.info;
  if (n_scans) *n_scans = (int)p.scans.size();
  for (int t = 0; scans && t < max_scans && t < (int)p.scans.size(); ++t) {
    const ibl::ScanInfo& si = p.scans[t];
    ibl_jpeg_scan& o = scans[t];
    o.components = si.ncomp;
    for (int i = 0; i < 3; ++i) o.comp[i] = i < si.ncomp ? si.comp[i] : -1;
    o.ss = si.ss;
    o.se = si.se;
    o.ah = si.ah;
    o.al = si.al;
    o.restart_interval = si.restart;
    o.intervals = si.n_iv;
  }
  if (st != IBL_OK) ibl::set_last_error(std::string("ibl_jpeg_parse_progressive: ") + p.info.reason);
  return st;
}
