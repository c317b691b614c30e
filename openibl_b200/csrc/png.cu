// PNG decode on the GPU, bit-identical to Pillow's `Image.open(f).convert('RGB')` (Preprocessor.__getitem__,
// ibl/utils/data/preprocessor.py:31-42) for 8-bit, non-interlaced PNGs of every colour type.  PNG is lossless, so
// "bit-identical" means a correct inflate and unfilter plus Pillow's mode conversion to RGB.
//
// Host: `parse_png` walks the chunks the way Pillow's PngImagePlugin does (CRCs verified before the first IDAT and
// not after it, the image data is the first run of IDAT chunks, IEND optional) and rejects, with a reason, everything
// Pillow would raise on, read differently, or that the device does not decode.  The IDAT payloads are concatenated
// into the engine's pinned staging blob, each stream followed by kPad zero bytes.
//
// Device, per batch (one pinned H2D copy, then two kernels on the caller's stream):
//   1. png_inflate_kernel   one warp per image inflates the whole zlib stream, following zlib's inflate.c and
//                           inftrees.c rules (over-subscribed codes and incomplete ones other than a single one-bit
//                           code are errors, a distance may reach back to the first byte produced whatever CINFO says,
//                           as non-strict zlib allows).  All 32 lanes run the Huffman decode in lockstep, so the
//                           decode state is uniform and a match is copied by all lanes at once into a 64 KiB ring in
//                           shared memory (the 32 KiB window plus the half being written); each completed half is
//                           stored to the row workspace [H][1 + W*bpp] with 16-byte coalesced stores and folded into
//                           the Adler-32.  Tables: a 10-bit (literal/length) and 8-bit (distance) primary table in
//                           shared memory; the rare longer codes are decoded canonically from the per-length counts.
//   2. png_unfilter_kernel  one block per image reverses the five scanline filters as a diagonal wavefront: thread r
//                           owns row r of a band of kRows rows and reconstructs pixel t - r at step t, with the pixel
//                           above handed over through shared memory; one barrier per step, W + rows - 1 steps per
//                           band.  It writes the RGB result straight into out_u8 (palette lookup, grey replicated,
//                           alpha dropped).
// Bounds: the bit reader clamps its load address to the stream's first kPad - 16 padding bytes and the decode stops
// as soon as it has consumed a bit past the stream; ring indices are masked; workspace stores are clipped to H rows;
// the unfilter reads only the workspace rows.  No input, however corrupt, reads or writes outside the buffers.
#include <string.h>

#include <algorithm>
#include <new>
#include <vector>

#include "common.cuh"

namespace ibl {

namespace {

constexpr int kPad = 32;             // zero bytes after every staged stream
constexpr int kLitRoot = 10;         // primary table bits, literal/length codes
constexpr int kDistRoot = 8;         // primary table bits, distance codes
constexpr int kClRoot = 7;           // code-length codes are at most 7 bits: all in the primary table
constexpr uint32_t kRingMask = 65535;
constexpr uint32_t kHalf = 32768;
constexpr int kRows = 256;           // unfilter band height (threads per block)
constexpr int kInflateSmem = 65536;  // the ring (dynamic shared memory)

// err_dev codes
enum { kErrData = 1, kErrShort = 2, kErrAdler = 3, kErrFilter = 4 };

struct PngImgDev {
  uint64_t z_off;       // stream in the blob's byte area (16-byte aligned)
  uint64_t z_len;       // stream bytes, zlib header included
  uint64_t ws_off;      // rows in the workspace (16-byte aligned)
  uint64_t out_off;     // RGB in out_u8
  uint32_t row_bytes;   // 1 + width * bpp
  int width, height, bpp, color_type, slot;
};

struct PngBatch {
  const PngImgDev* img;
  const uint8_t* pal;   // [M][768], zero past the PLTE entries
  const uint8_t* bytes;
  uint8_t* ws;
  uint8_t* out;
  int* err;
};

__constant__ uint16_t c_lbase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                     31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                     193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// LSB-first bit reader over one staged stream.  Invariant: bits [0, nb) of bb are the stream's bits from
// consumed() on, and the bits above them are the following stream bytes, so OR-ing a fresh load is idempotent.
struct Bits {
  const uint8_t* src;
  uint64_t len;
  uint64_t bb;
  uint64_t pos;   // next byte to load
  int nb;
  __device__ __forceinline__ void refill() {
    // a read past the stream only happens once the decode has consumed a bit past it (and stops): clamping keeps
    // both 8-byte loads inside the stream's padding (len + 8 + 16 <= len + kPad)
    const uint64_t p = pos < len + 8 ? pos : len + 8;
    const uint64_t a = p & ~7ull;
    const int sh = (int)(p & 7) * 8;
    const uint64_t lo = *reinterpret_cast<const uint64_t*>(src + a);
    const uint64_t hi = *reinterpret_cast<const uint64_t*>(src + a + 8);
    const uint64_t w = sh ? (lo >> sh) | (hi << (64 - sh)) : lo;
    bb |= w << nb;
    pos += (63 - nb) >> 3;
    nb |= 56;
  }
  __device__ __forceinline__ uint32_t take(int n) {
    const uint32_t v = (uint32_t)(bb & ((1ull << n) - 1));
    bb >>= n;
    nb -= n;
    return v;
  }
  __device__ __forceinline__ uint64_t consumed() const { return pos * 8 - nb; }
  __device__ __forceinline__ bool over() const { return consumed() > len * 8; }
};

// A canonical Huffman code in shared memory: primary table entries are sym | len << 9 (0 = longer code or no code),
// count[len] and the symbols sorted by (len, sym) serve the codes longer than the root.
struct Code {
  uint16_t* tab;
  uint16_t* count;
  uint16_t* sorted;
  int root;
};

// Builds `c` from n code lengths.  Returns 0 for a complete code, 1 for an incomplete one with codes longer than one
// bit, 2 for no codes at all, 3 for a single one-bit code and -1 for an over-subscribed one (inftrees.c's cases).
__device__ int build_code(const uint8_t* lens, int n, Code c, uint16_t* codes, int* res, int lane) {
  if (lane == 0) {
    for (int l = 0; l < 16; ++l) c.count[l] = 0;
    for (int s = 0; s < n; ++s) c.count[lens[s]]++;
    c.count[0] = 0;
    int left = 1, maxl = 0;
    for (int l = 1; l < 16; ++l) {
      left = (left << 1) - c.count[l];
      if (left < 0) break;
      if (c.count[l]) maxl = l;
    }
    int r;
    if (left < 0) r = -1;
    else if (left == 0) r = 0;
    else r = maxl == 0 ? 2 : (maxl == 1 ? 3 : 1);
    if (r >= 0) {
      uint16_t next[16], offs[16];
      int code = 0, off = 0;
      for (int l = 1; l < 16; ++l) {
        code = (code + (l > 1 ? c.count[l - 1] : 0)) << 1;
        next[l] = (uint16_t)code;
        offs[l] = (uint16_t)off;
        off += c.count[l];
      }
      for (int s = 0; s < n; ++s) {
        const int l = lens[s];
        if (l) {
          codes[s] = next[l]++;
          c.sorted[offs[l]++] = (uint16_t)s;
        }
      }
    }
    *res = r;
  }
  for (int e = lane; e < (1 << c.root); e += 32) c.tab[e] = 0;
  __syncwarp();
  const int r = *res;
  if (r >= 0) {
    for (int s = lane; s < n; s += 32) {
      const int l = lens[s];
      if (l && l <= c.root) {
        const int rev = (int)(__brev((unsigned)codes[s]) >> (32 - l));
        for (int e = rev; e < (1 << c.root); e += 1 << l) c.tab[e] = (uint16_t)(s | (l << 9));
      }
    }
  }
  __syncwarp();
  return r;
}

// Next symbol, or -1 for a bit pattern that is no code (nothing consumed then).  Needs 15 valid bits.
__device__ __forceinline__ int decode_sym(Bits& br, const Code& c) {
  const uint16_t e = c.tab[br.bb & ((1u << c.root) - 1)];
  if (e) {
    br.bb >>= (e >> 9);
    br.nb -= (e >> 9);
    return e & 511;
  }
  int code = 0, first = 0, index = 0;
  for (int l = 1; l < 16; ++l) {
    code |= (int)((br.bb >> (l - 1)) & 1);
    const int cnt = c.count[l];
    if (code - cnt < first) {
      br.bb >>= l;
      br.nb -= l;
      return c.sorted[index + code - first];
    }
    index += cnt;
    first = (first + cnt) << 1;
    code <<= 1;
  }
  return -1;
}

// Stores ring bytes [from, from + n) (n <= kHalf, `from` a multiple of kHalf) to the workspace, clipped to the rows,
// and folds them into the Adler-32 (a, b).
__device__ void flush(const uint8_t* ring, uint8_t* dst, uint64_t rows_total, uint64_t from, uint32_t n, uint32_t& a,
                      uint32_t& b, int lane) {
  __syncwarp();
  const uint8_t* r = ring + (from & kRingMask);
  uint32_t s = 0;
  uint64_t w = 0;
  const uint32_t n16 = n & ~15u;
  for (uint32_t j = lane * 16; j < n16; j += 512) {
    const uint4 q = *reinterpret_cast<const uint4*>(r + j);
    const uint64_t g = from + j;
    if (g + 16 <= rows_total) {
      *reinterpret_cast<uint4*>(dst + g) = q;
    } else {
      for (uint32_t k = 0; g + k < rows_total && k < 16; ++k) dst[g + k] = r[j + k];
    }
    const uint32_t v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const uint32_t byte = (v[k >> 2] >> (8 * (k & 3))) & 255;
      s += byte;
      w += (uint64_t)(n - j - k) * byte;
    }
  }
  for (uint32_t j = n16 + lane; j < n; j += 32) {
    const uint32_t byte = r[j];
    if (from + j < rows_total) dst[from + j] = (uint8_t)byte;
    s += byte;
    w += (uint64_t)(n - j) * byte;
  }
  uint64_t s64 = s;
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    s64 += __shfl_xor_sync(0xffffffffu, s64, o);
    w += __shfl_xor_sync(0xffffffffu, w, o);
  }
  const uint32_t a0 = a;
  a = (uint32_t)((a0 + s64 % 65521) % 65521);
  b = (uint32_t)((b + (uint64_t)(n % 65521) * a0 + w % 65521) % 65521);
  __syncwarp();
}

__global__ void __launch_bounds__(32) png_inflate_kernel(PngBatch bt) {
  extern __shared__ __align__(16) uint8_t ring[];
  __shared__ uint16_t lit_tab[1 << kLitRoot], dist_tab[1 << kDistRoot], cl_tab[1 << kClRoot];
  __shared__ uint16_t lit_count[16], dist_count[16], cl_count[16];
  __shared__ uint16_t lit_sorted[288], dist_sorted[32], cl_sorted[19], codes[320];
  __shared__ uint8_t lens[320];
  __shared__ int res;
  const PngImgDev im = bt.img[blockIdx.x];
  const int lane = threadIdx.x;
  const Code lit{lit_tab, lit_count, lit_sorted, kLitRoot}, dist{dist_tab, dist_count, dist_sorted, kDistRoot},
      cl{cl_tab, cl_count, cl_sorted, kClRoot};
  uint8_t* dst = bt.ws + im.ws_off;
  const uint64_t rows_total = (uint64_t)im.height * im.row_bytes;
  Bits br{bt.bytes + im.z_off, im.z_len, 0, 2, 0};   // past the zlib header, which the parse validated
  uint64_t P = 0, flushed = 0;                       // bytes produced / already stored
  uint32_t ad_a = 1, ad_b = 0;
  int state = 0;                                     // 1 final block done, 2 input ran out, 3 corrupt data
  while (state == 0) {
    br.refill();
    const uint32_t hdr = br.take(3);
    if (br.over()) { state = 2; break; }
    const int type = (int)(hdr >> 1);
    if (type == 0) {                                 // stored
      br.take(br.nb & 7);
      br.refill();
      const uint32_t ln = br.take(16), nl = br.take(16);
      if (br.over()) { state = 2; break; }
      if ((ln ^ 0xFFFFu) != nl) { state = 3; break; }
      const uint64_t bp = br.consumed() >> 3;
      const uint32_t n = (uint32_t)std::min<uint64_t>(ln, im.z_len - bp);
      for (uint32_t done = 0; done < n;) {
        const uint32_t c = std::min<uint32_t>(n - done, (uint32_t)(flushed + kHalf - P));
        for (uint32_t i = lane; i < c; i += 32) ring[(P + i) & kRingMask] = br.src[bp + done + i];
        P += c;
        done += c;
        if (P - flushed >= kHalf) {
          flush(ring, dst, rows_total, flushed, kHalf, ad_a, ad_b, lane);
          flushed += kHalf;
        }
      }
      br.pos = bp + n;
      br.bb = 0;
      br.nb = 0;
      if (n < ln) { state = 2; break; }
    } else if (type == 3) {
      state = 3;
      break;
    } else {
      int hlit = 288, hdist = 30;
      if (type == 1) {                               // fixed codes; literal 286/287 and distance 30/31 are invalid
        for (int s = lane; s < 318; s += 32)
          lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
        __syncwarp();
      } else {                                       // dynamic: the code-length code, then the code lengths
        br.refill();
        hlit = (int)br.take(5) + 257;
        hdist = (int)br.take(5) + 1;
        const int hclen = (int)br.take(4) + 4;
        if (br.over()) { state = 2; break; }
        if (hlit > 286 || hdist > 30) { state = 3; break; }
        uint8_t* cll = lens + 288;                   // 19 code-length code lengths, clear of lens[0..288)
        for (int k0 = 0; k0 < 19; k0 += 10) {        // 3 bits each, at most 30 per refill
          br.refill();
          const int k = k0 + lane, cnt = std::max(0, std::min(10, hclen - k0));
          if (lane < 10 && k < 19) cll[c_clorder[k]] = k < hclen ? (uint8_t)((br.bb >> (3 * lane)) & 7) : 0;
          br.take(3 * cnt);
        }
        if (br.over()) { state = 2; break; }
        __syncwarp();
        if (build_code(cll, 19, cl, codes, &res, lane) != 0) { state = 3; break; }
        // the lengths go to lens[0..hlit+hdist) (<= 316), overwriting cll only after it has been used for the table
        int n = 0;
        while (n < hlit + hdist) {
          br.refill();
          const int sym = decode_sym(br, cl);
          if (sym < 0) { state = 3; break; }         // cannot happen: the code is complete
          int rep = 1, val = sym;
          if (sym == 16) {
            if (n == 0) { state = br.over() ? 2 : 3; break; }
            rep = 3 + (int)br.take(2);
            val = lens[n - 1];
          } else if (sym == 17) {
            rep = 3 + (int)br.take(3);
            val = 0;
          } else if (sym == 18) {
            rep = 11 + (int)br.take(7);
            val = 0;
          }
          if (br.over()) { state = 2; break; }
          if (n + rep > hlit + hdist) { state = 3; break; }
          __syncwarp();
          for (int i = lane; i < rep; i += 32) lens[n + i] = (uint8_t)val;
          n += rep;
          __syncwarp();
        }
        if (state) break;
        if (lens[256] == 0) { state = 3; break; }
      }
      const int rl = build_code(lens, hlit, lit, codes, &res, lane);
      const int rd = build_code(lens + hlit, hdist, dist, codes, &res, lane);
      if (type == 2 && (rl < 0 || rl == 1 || rd < 0 || rd == 1)) { state = 3; break; }
      for (;;) {
        if (br.nb < 48) br.refill();                 // a literal/length and a distance take at most 48 bits
        const int sym = decode_sym(br, lit);
        if (sym < 0 || sym >= 286) { state = br.consumed() + 15 > br.len * 8 ? 2 : 3; break; }
        if (sym < 256) {
          if (br.over()) { state = 2; break; }
          if (lane == 0) ring[P & kRingMask] = (uint8_t)sym;
          ++P;
        } else if (sym == 256) {
          if (br.over()) state = 2;
          break;
        } else {
          const int li = sym - 257;
          const uint32_t len = c_lbase[li] + br.take(c_lext[li]);
          const int ds = decode_sym(br, dist);
          if (ds < 0 || ds >= 30) { state = br.consumed() + 15 > br.len * 8 ? 2 : 3; break; }
          const uint32_t d = c_dbase[ds] + br.take(c_dext[ds]);
          if (br.over()) { state = 2; break; }
          if (d > P) { state = 3; break; }
          __syncwarp();
          // byte i of the match repeats byte i mod d of the d bytes before it, all of which are already in the ring
          for (uint32_t i = lane; i < len; i += 32)
            ring[(P + i) & kRingMask] = ring[(P - d + (i < d ? i : i % d)) & kRingMask];
          P += len;
        }
        if (P - flushed >= kHalf) {                  // at most kHalf + 257 bytes unflushed: the ring holds them
          flush(ring, dst, rows_total, flushed, kHalf, ad_a, ad_b, lane);
          flushed += kHalf;
        }
      }
    }
    if (state == 0 && (hdr & 1)) state = 1;
  }
  if (P > flushed) flush(ring, dst, rows_total, flushed, (uint32_t)(P - flushed), ad_a, ad_b, lane);
  int err = 0;
  if (state == 3) {
    err = kErrData;
  } else if (P < rows_total) {
    err = kErrShort;
  } else if (state == 1) {                           // the Adler-32 is checked when the stream carries all of it
    br.take(br.nb & 7);
    br.refill();
    if ((br.consumed() >> 3) + 4 <= br.len) {
      uint32_t want = 0;
      for (int k = 0; k < 4; ++k) want = (want << 8) | br.take(8);
      if (want != ((ad_b << 16) | ad_a)) err = kErrAdler;
    }
  }
  if (err && lane == 0) bt.err[im.slot] = err;
}

__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__global__ void __launch_bounds__(kRows) png_unfilter_kernel(PngBatch bt) {
  __shared__ uint32_t up_px[2][kRows];               // the pixel each row reconstructed at the last two steps
  __shared__ uint8_t pal[768];
  const PngImgDev im = bt.img[blockIdx.x];
  const int tid = threadIdx.x;
  if (im.color_type == 3)
    for (int i = tid; i < 768; i += kRows) pal[i] = bt.pal[(size_t)blockIdx.x * 768 + i];
  const int W = im.width, bpp = im.bpp;
  uint8_t* ws = bt.ws + im.ws_off;
  uint8_t* out = bt.out + im.out_off;
  bool bad = false;
  for (int r0 = 0; r0 < im.height; r0 += kRows) {
    const int rows = im.height - r0 < kRows ? im.height - r0 : kRows, r = r0 + tid;
    const bool active = tid < rows;
    uint8_t* row = ws + (size_t)r * im.row_bytes;
    int ft = active ? row[0] : 0;
    if (ft > 4) {
      bad = true;
      ft = 0;
    }
    const uint8_t* above = r > 0 ? row - im.row_bytes : nullptr;   // read by thread 0 only: the previous band's last row
    uint32_t left = 0, upleft = 0;
    __syncthreads();                                 // the previous band's last row is stored
    for (int t = 0; t < W + rows - 1; ++t) {
      const int x = t - tid;
      if (active && x >= 0 && x < W) {
        uint32_t up = 0;
        if (tid > 0) {
          up = up_px[(t - 1) & 1][tid - 1];
        } else if (above) {
          for (int k = 0; k < bpp; ++k) up |= (uint32_t)above[1 + x * bpp + k] << (8 * k);
        }
        const uint8_t* p = row + 1 + x * bpp;
        uint32_t px = 0;
        for (int k = 0; k < bpp; ++k) {
          const int a = (left >> (8 * k)) & 255, b = (up >> (8 * k)) & 255, c = (upleft >> (8 * k)) & 255;
          int v = p[k];
          if (ft == 1) v += a;
          else if (ft == 2) v += b;
          else if (ft == 3) v += (a + b) >> 1;
          else if (ft == 4) v += paeth(a, b, c);
          px |= (uint32_t)(v & 255) << (8 * k);
        }
        up_px[t & 1][tid] = px;
        if (tid == rows - 1)                         // the next band's first row reads it from the workspace
          for (int k = 0; k < bpp; ++k) row[1 + x * bpp + k] = (uint8_t)(px >> (8 * k));
        left = px;
        upleft = up;
        uint8_t* o = out + ((size_t)r * W + x) * 3;
        if (im.color_type == 3) {
          const int i = px & 255;
          o[0] = pal[3 * i];
          o[1] = pal[3 * i + 1];
          o[2] = pal[3 * i + 2];
        } else if (im.color_type == 0 || im.color_type == 4) {
          o[0] = o[1] = o[2] = (uint8_t)px;
        } else {
          o[0] = (uint8_t)px;
          o[1] = (uint8_t)(px >> 8);
          o[2] = (uint8_t)(px >> 16);
        }
      }
      __syncthreads();
    }
  }
  if (bad) bt.err[im.slot] = kErrFilter;
}

// ---- host: chunk walk -----------------------------------------------------------------------------------------------

struct Crc32 {
  uint32_t t[256];
  Crc32() {
    for (uint32_t n = 0; n < 256; ++n) {
      uint32_t c = n;
      for (int k = 0; k < 8; ++k) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
      t[n] = c;
    }
  }
  uint32_t operator()(const uint8_t* p, size_t n) const {
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; ++i) c = t[(c ^ p[i]) & 255] ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
  }
};
const Crc32 crc32;

struct PngParsed {
  ibl_png_info info;
  std::vector<std::pair<size_t, size_t>> idat;   // (file offset, bytes) of the stream's pieces
  uint8_t plte[768];
};

uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

bool is_cid(const uint8_t* id) {   // Pillow's re.match(rb"\w\w\w\w")
  for (int k = 0; k < 4; ++k) {
    const uint8_t c = id[k];
    if (!((c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_')) return false;
  }
  return true;
}

int bpp_of(int ct) { return ct == 2 ? 3 : ct == 4 ? 2 : ct == 6 ? 4 : 1; }

// Chunks whose Pillow handler could raise or change how the pixels are read: accepted when `len` is what the handler
// needs, rejected (reason) otherwise.  Chunks Pillow has no handler for are skipped, as Pillow skips them.
const char* chunk_problem(const uint8_t* id, uint32_t len, int ct, bool after_idat) {
  auto is = [&](const char* s) { return memcmp(id, s, 4) == 0; };
  if (is("IHDR")) return after_idat ? "IHDR after IDAT" : "second IHDR";
  if (is("PLTE")) return after_idat ? "PLTE after IDAT" : nullptr;
  if (is("tRNS")) {
    if (after_idat) return "tRNS after IDAT";
    if ((ct == 0 && len < 2) || (ct == 2 && len < 6)) return "short tRNS";
    return nullptr;
  }
  if (is("gAMA")) return len < 4 ? "short gAMA" : nullptr;
  if (is("cHRM")) return len % 4 ? "cHRM length not a multiple of 4" : nullptr;
  if (is("sRGB")) return len < 1 ? "short sRGB" : nullptr;
  if (is("pHYs")) return len < 9 ? "short pHYs" : nullptr;
  if (is("iCCP") || is("zTXt") || is("iTXt")) return "compressed ancillary chunk (iCCP/zTXt/iTXt)";
  if (is("acTL") || is("fcTL") || is("fdAT")) return "APNG";
  if (is("IDAT") || is("DDAT")) return "IDAT after other chunks";
  return nullptr;
}

int parse_png(const uint8_t* d, size_t n, PngParsed& p) {
  memset(&p.info, 0, sizeof(p.info));
  memset(p.plte, 0, sizeof(p.plte));
  p.idat.clear();
  ibl_png_info& info = p.info;
  auto reject = [&](const char* why) {
    snprintf(info.reason, sizeof(info.reason), "%s", why);
    return IBL_ERR_UNSUPPORTED;
  };
  static const uint8_t sig[8] = {137, 80, 78, 71, 13, 10, 26, 10};
  if (!d || n < 8 || memcmp(d, sig, 8) != 0) return reject("not a PNG file");
  size_t pos = 8;
  bool have_ihdr = false, have_plte = false;
  int ct = -1;
  // before the first IDAT: every chunk complete, CRC verified (ChunkStream.crc)
  for (;;) {
    if (n - pos < 8) return reject("file ends before IDAT");
    const uint32_t len = be32(d + pos);
    const uint8_t* id = d + pos + 4;
    if (!is_cid(id)) return reject("bad chunk type");
    if (!have_ihdr && memcmp(id, "IHDR", 4) != 0) return reject("IHDR is not the first chunk");
    if (memcmp(id, "IDAT", 4) == 0) break;
    if (n - pos - 8 < (size_t)len + 4) return reject("chunk cut short before IDAT");
    if (crc32(id, (size_t)len + 4) != be32(d + pos + 8 + len)) return reject("bad CRC before IDAT");
    const uint8_t* s = d + pos + 8;
    if (memcmp(id, "IEND", 4) == 0) return reject("no IDAT");
    if (!have_ihdr) {
      if (len != 13) return reject("IHDR length is not 13");
      info.width = (int)std::min<uint32_t>(be32(s), 0x7FFFFFFF);
      info.height = (int)std::min<uint32_t>(be32(s + 4), 0x7FFFFFFF);
      info.bit_depth = s[8];
      info.color_type = ct = s[9];
      if (s[11] != 0) return reject("unknown filter method");
      if (ct != 0 && ct != 2 && ct != 3 && ct != 4 && ct != 6) return reject("unknown colour type");
      if (info.bit_depth != 8) return reject("bit depth is not 8");
      if (s[12] != 0) return reject("interlaced");
      if (info.width == 0 || info.height == 0) return reject("zero width or height");
      if ((uint64_t)info.width * info.height > 89478485ull) return reject("more pixels than Pillow's MAX_IMAGE_PIXELS");
      have_ihdr = true;
    } else {
      if (const char* why = chunk_problem(id, len, ct, false)) return reject(why);
      if (memcmp(id, "PLTE", 4) == 0) {
        if (have_plte) return reject("second PLTE");
        if (len == 0 || len % 3 != 0 || len > 768) return reject("bad PLTE length");
        if (ct == 3) {
          memcpy(p.plte, s, len);
          info.palette_size = (int)(len / 3);
        }
        have_plte = true;
      }
    }
    pos += 12 + (size_t)len;
  }
  if (ct == 3 && info.palette_size == 0) return reject("palette image without PLTE");
  // the first run of IDAT chunks is the stream (PngImageFile.load_read); the file may end inside it
  uint64_t zlen = 0;
  while (n - pos >= 8 && memcmp(d + pos + 4, "IDAT", 4) == 0) {
    const uint32_t len = be32(d + pos);
    const size_t avail = std::min<size_t>(len, n - pos - 8);
    if (avail) p.idat.emplace_back(pos + 8, avail);
    zlen += avail;
    if (avail < len || n - pos - 8 - len < 4) {
      pos = n;
      break;
    }
    pos += 12 + (size_t)len;
  }
  // after it (PngImageFile.load_end): handlers run up to IEND, CRCs are not checked, a short chunk raises
  while (n - pos >= 8 && is_cid(d + pos + 4) && memcmp(d + pos + 4, "IEND", 4) != 0) {
    const uint32_t len = be32(d + pos);
    if (n - pos - 8 < len) return reject("chunk cut short after IDAT");
    if (const char* why = chunk_problem(d + pos + 4, len, ct, true)) return reject(why);
    pos += 8 + (size_t)len + std::min<size_t>(4, n - pos - 8 - len);
  }
  info.zlib_bytes = zlen;
  if (zlen < 2) return reject("no zlib header");
  uint8_t h[2];
  {
    int k = 0;
    for (const auto& pc : p.idat)
      for (size_t i = 0; i < pc.second && k < 2; ++i) h[k++] = d[pc.first + i];
  }
  if ((h[0] & 15) != 8) return reject("zlib method is not deflate");
  if ((h[0] >> 4) > 7) return reject("zlib window larger than 32 KiB");
  if (((unsigned)h[0] << 8 | h[1]) % 31 != 0) return reject("bad zlib header check");
  if (h[1] & 0x20) return reject("zlib preset dictionary");
  return IBL_OK;
}

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

}  // namespace

int png_decode_u8(JpegWs** pws, const uint8_t* const* files, const size_t* lens, int N, uint8_t* out_u8,
                  const uint64_t* out_offsets, int* status, int* err_dev, cudaStream_t s, uint64_t* launches) {
  IBL_RET(ws_open(pws));
  JpegWs* ws = *pws;
  IBL_CUDA_OK(cudaMemsetAsync(err_dev, 0, (size_t)N * sizeof(int), s));
  std::vector<PngParsed> ps;
  std::vector<int> slot;
  for (int i = 0; i < N; ++i) {
    PngParsed p;
    status[i] = files[i] ? parse_png(files[i], lens[i], p) : IBL_ERR_BAD_ARG;
    if (status[i] != IBL_OK) continue;
    ps.push_back(std::move(p));
    slot.push_back(i);
  }
  const int M = (int)ps.size();
  if (M == 0) return IBL_OK;
  std::vector<PngImgDev> imgs(M);
  uint64_t zbytes = 0, wbytes = 0;
  for (int m = 0; m < M; ++m) {
    const ibl_png_info& inf = ps[m].info;
    PngImgDev& im = imgs[m];
    im.width = inf.width;
    im.height = inf.height;
    im.color_type = inf.color_type;
    im.bpp = bpp_of(inf.color_type);
    im.row_bytes = 1u + (uint32_t)inf.width * im.bpp;
    im.slot = slot[m];
    im.out_off = out_offsets[slot[m]];
    im.z_off = zbytes;
    im.z_len = inf.zlib_bytes;
    zbytes += align16(inf.zlib_bytes + kPad);
    im.ws_off = wbytes;
    wbytes += align16((uint64_t)im.height * im.row_bytes);
  }
  // staging blob: images | palettes | streams (each zero-padded)
  const size_t o_img = 0, o_pal = align16(sizeof(PngImgDev) * M), o_bytes = align16(o_pal + 768 * (size_t)M),
               blob_bytes = o_bytes + zbytes;
  IBL_RET(stage_host(ws, blob_bytes));
  uint8_t* h = ws->host;
  memcpy(h + o_img, imgs.data(), sizeof(PngImgDev) * M);
  for (int m = 0; m < M; ++m) {
    memcpy(h + o_pal + 768 * (size_t)m, ps[m].plte, 768);
    uint8_t* z = h + o_bytes + imgs[m].z_off;
    for (const auto& pc : ps[m].idat) {
      memcpy(z, files[slot[m]] + pc.first, pc.second);
      z += pc.second;
    }
    memset(z, 0, align16(imgs[m].z_len + kPad) - imgs[m].z_len);
  }
  IBL_RET(grow_device(&ws->blob, &ws->blob_cap, blob_bytes));
  IBL_RET(grow_device(&ws->arena, &ws->arena_cap, std::max<uint64_t>(wbytes, 16)));
  IBL_CUDA_OK(cudaMemcpyAsync(ws->blob, ws->host, blob_bytes, cudaMemcpyHostToDevice, s));
  IBL_CUDA_OK(cudaEventRecord(ws->copied, s));
  ws->pending = true;
  const uint8_t* db = static_cast<const uint8_t*>(ws->blob);
  PngBatch b;
  b.img = reinterpret_cast<const PngImgDev*>(db + o_img);
  b.pal = db + o_pal;
  b.bytes = db + o_bytes;
  b.ws = static_cast<uint8_t*>(ws->arena);
  b.out = out_u8;
  b.err = err_dev;
  static DeviceOnce attr;
  if (!attr.done()) {
    IBL_CUDA_OK(cudaFuncSetAttribute(png_inflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kInflateSmem));
    attr.mark();
  }
  png_inflate_kernel<<<M, 32, kInflateSmem, s>>>(b);
  png_unfilter_kernel<<<M, kRows, 0, s>>>(b);
  IBL_CUDA_OK(cudaGetLastError());
  if (launches) *launches += 2;
  return IBL_OK;
}

}  // namespace ibl

extern "C" int ibl_png_parse(const uint8_t* data, size_t len, ibl_png_info* out) {
  IBL_REQUIRE(out, "null argument");
  ibl::PngParsed p;
  const int st = ibl::parse_png(data, len, p);
  *out = p.info;
  if (st != IBL_OK) ibl::set_last_error(std::string("ibl_png_parse: ") + p.info.reason);
  return st;
}
