// Baseline JPEG decode for the device presets, bit-identical to PIL's decode through libjpeg-turbo:
//   * hk_jpeg_huffman: the entropy decode of every image's scan, in parallel by self-synchronisation (Weissenberger &
//     Schmidt, "Massively Parallel Huffman Decoding on GPUs", ICPP 2018).  The scan of each restart segment is cut into
//     chunks; a thread decodes its chunk from an entry state (bit position, block of the MCU, zig-zag index) and records
//     the state it reaches at the chunk's end as its successor's entry.  A chunk whose entry changed is decoded again,
//     until no entry changes.  The first chunk of a segment starts from the exact state, so by induction every entry
//     is then exact whatever was guessed: a slow synchronisation costs iterations, never a wrong coefficient.  Block
//     counts and DC differences per chunk are prefix-summed over the image, and a last pass writes the coefficients,
//     de-zig-zagged, with the DC values absolute.
//   * hk_jpeg_idct: dequantisation and jpeg_idct_islow (jidctint.c) with its range limiting, one thread per block.
//   * hk_jpeg_color: jdsample.c's fancy upsampling (h2v1, h2v2: the triangle filters, their edge columns and rows,
//     their alternating rounding) and jdcolor.c's YCbCr -> RGB tables, written cropped into the pixel buffer.
// hawkeye_b200/ops_jpeg.py parses the markers on the host and lays out the tables; tests/jpeg_ref.py restates the
// arithmetic.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

// columns of the per-image header (ops_jpeg.py H_*)
enum JpegCol {
  JC_IMG, JC_W, JC_H, JC_NCOMP, JC_HY, JC_VY, JC_MCUX, JC_MCUY, JC_RI, JC_SEG0, JC_NSEG, JC_BLK0, JC_PLANE0,
  JC_Q0, JC_DC0 = JC_Q0 + 3, JC_AC0 = JC_DC0 + 3, JPEG_COLS = JC_AC0 + 3
};

enum JpegStatus { JS_OK, JS_BAD_CODE, JS_ENDS_EARLY, JS_TRAILING, JS_SEGMENTS, JS_INDEX };

constexpr int LOOK_BITS = 9;

// a DHT in the form the decoder reads (ops_jpeg.py HTAB_DTYPE): maxcode[l] / valoffset[l] for code length l of 1..16
// (maxcode -1 where no code has that length), the symbols, and (length << 8 | symbol) for every 9-bit prefix whose
// code is at most 9 bits long, 0 otherwise
struct HuffTab {
  int maxcode[18];
  int valoffset[18];
  unsigned char huffval[256];
  unsigned short look[1 << LOOK_BITS];
};
static_assert(sizeof(HuffTab) == 1424, "HuffTab layout");

__constant__ unsigned char kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                           12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                           35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                           58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// decoder state at a symbol boundary: bit position, block of the MCU, zig-zag index
__device__ __forceinline__ unsigned long long pack_state(uint32_t p, int b, int k) {
  return (unsigned long long)p | ((unsigned long long)b << 32) | ((unsigned long long)k << 40);
}

constexpr int HUFF_THREADS = 512;

struct ImgTabs {
  HuffTab t[6];      // DC, AC of each component
  int ny, bpm;       // luma blocks and blocks per MCU
};

// the 32 bits of the scan from bit p on (MSB first); the scan is padded so that p + 64 bits stay inside
__device__ __forceinline__ uint32_t peek32(const uint32_t* __restrict__ words, uint32_t p) {
  const uint32_t w = p >> 5;
  const unsigned long long hi = __byte_perm(words[w], 0, 0x0123), lo = __byte_perm(words[w + 1], 0, 0x0123);
  return (uint32_t)((((hi << 32) | lo) << (p & 31)) >> 32);
}

// One Huffman symbol at bit p of block b of the MCU at zig-zag index k (libjpeg's decode_mcu): advances p, b, k.  The
// symbol covers zig-zag positions [k, kend) with value `val` at `pos` (-1: none) and zeros elsewhere; `done` when it
// ends its block.  -> 0 or a JpegStatus.
__device__ __forceinline__ int jpeg_symbol(const ImgTabs& it, const uint32_t* __restrict__ words, uint32_t& p, int& b,
                                           int& k, int& pos, int& val, int& kend, bool& done) {
  const uint32_t win = peek32(words, p);
  const int comp = b < it.ny ? 0 : b - it.ny + 1;
  const HuffTab& t = it.t[2 * comp + (k != 0)];
  int len = 0, sym = 0;
  const int e = t.look[win >> (32 - LOOK_BITS)];
  if (e) {
    len = e >> 8;
    sym = e & 255;
  } else {
    for (int l = LOOK_BITS + 1; l <= 16; ++l) {
      const int code = (int)(win >> (32 - l));
      if (code <= t.maxcode[l]) {
        len = l;
        sym = t.huffval[(code + t.valoffset[l]) & 255];
        break;
      }
    }
    if (!len) return JS_BAD_CODE;
  }
  const int s = k == 0 ? sym : (sym & 15), r = k == 0 ? 0 : (sym >> 4);
  int v = 0;
  if (s) {
    v = (int)((win << len) >> (32 - s));
    if (v < (1 << (s - 1))) v -= (1 << s) - 1;
  }
  p += len + s;
  pos = -1;
  val = v;
  if (k == 0) {
    pos = 0;
    k = 1;
  } else if (s) {
    k += r;
    if (k > 63) return JS_INDEX;
    pos = k++;
  } else if (r == 15) {
    k += 16;
    if (k > 64) return JS_INDEX;
  } else {
    k = 64;
  }
  kend = k;
  done = k == 64;
  if (done) {
    k = 0;
    if (++b == it.bpm) b = 0;
  }
  return JS_OK;
}

// workspace of the Huffman pass: per segment (plus one per image) the first chunk; per chunk the entry state, the state
// its predecessor reached, a dirty flag, its segment and its (blocks, DC sum per component)
struct HuffWs {
  int* seg_chunk;
  unsigned long long *entry, *reached;
  int *dirty, *seg, *cnt;          // cnt: 4 ints per chunk
};

__host__ __device__ inline long long huff_chunks_bound(int J, int G, long long scan_bytes, int chunk) {
  return scan_bytes / chunk + G + 2LL * J + 2;
}

__host__ __device__ inline HuffWs huff_ws(void* base, int J, int G, long long nch) {
  HuffWs w;
  char* p = (char*)base;
  w.entry = (unsigned long long*)p;
  p += nch * 8;
  w.reached = (unsigned long long*)p;
  p += nch * 8;
  w.cnt = (int*)p;
  p += nch * 16;
  w.dirty = (int*)p;
  p += nch * 4;
  w.seg = (int*)p;
  p += nch * 4;
  w.seg_chunk = (int*)p;
  return w;
}

__host__ __device__ inline size_t huff_ws_bytes(int J, int G, long long nch) {
  return (size_t)nch * 40 + (size_t)(G + J) * 4;
}

// One CTA per image: the chunk layout, the synchronisation loop, the prefix sums and the coefficient pass.
__global__ void __launch_bounds__(HUFF_THREADS) jpeg_huffman_kernel(
    const uint32_t* __restrict__ words, const int* __restrict__ segs, const int* __restrict__ header,
    const HuffTab* __restrict__ htabs, short* __restrict__ coef, int* __restrict__ status, int chunk, HuffWs ws) {
  __shared__ ImgTabs it;
  __shared__ int red[32];
  __shared__ int s_status, s_done, s_first_err;
  const int j = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int* h = header + (size_t)j * JPEG_COLS;
  const int ncomp = h[JC_NCOMP], hy = h[JC_HY], vy = h[JC_VY], mcux = h[JC_MCUX], mcuy = h[JC_MCUY];
  const int seg0 = h[JC_SEG0], nseg = h[JC_NSEG];
  const int total_mcus = mcux * mcuy, ri = h[JC_RI] > 0 ? h[JC_RI] : total_mcus;
  if (tid == 0) {
    it.ny = hy * vy;
    it.bpm = hy * vy + ncomp - 1;
    s_status = nseg == (total_mcus + ri - 1) / ri ? JS_OK : JS_SEGMENTS;
    s_done = 0;
    s_first_err = INT_MAX;
  }
  for (int c = 0; c < ncomp; ++c)
    for (int i = tid; i < (int)(sizeof(HuffTab) / 4); i += nt) {
      ((int*)&it.t[2 * c])[i] = ((const int*)(htabs + h[JC_DC0 + c]))[i];
      ((int*)&it.t[2 * c + 1])[i] = ((const int*)(htabs + h[JC_AC0 + c]))[i];
    }
  __syncthreads();
  if (s_status != JS_OK) {
    if (tid == 0) status[j] = s_status;
    return;
  }
  const int bpm = it.bpm;
  // the chunks of each segment: max(1, ceil(bytes / chunk)), laid out segment after segment
  int* seg_chunk = ws.seg_chunk + seg0 + j;
  const long long cbase = segs[seg0] / chunk + seg0 + 2LL * j;
  unsigned long long* entry = ws.entry + cbase;
  unsigned long long* reached = ws.reached + cbase;
  int* dirty = ws.dirty + cbase;
  int* cseg = ws.seg + cbase;
  int4* cnt = (int4*)ws.cnt + cbase;
  int carry = 0;
  for (int s0 = 0; s0 < nseg; s0 += nt) {
    const int s = s0 + tid;
    int n = 0;
    if (s < nseg) {
      const int bytes = segs[seg0 + s + 1] - segs[seg0 + s];
      n = bytes > 0 ? (bytes + chunk - 1) / chunk : 1;
    }
    int tile;
    const int ex = block_exclusive_scan(n, red, tile);
    if (s < nseg) seg_chunk[s] = carry + ex;
    carry += tile;
  }
  const int nch = carry;
  if (tid == 0) seg_chunk[nseg] = nch;
  __syncthreads();
  for (int i = tid; i < nch; i += nt) {
    int lo = 0, hi = nseg - 1;                      // the last segment whose first chunk is <= i
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (seg_chunk[mid] <= i) lo = mid;
      else hi = mid - 1;
    }
    cseg[i] = lo;
    const uint32_t start = (uint32_t)(segs[seg0 + lo] + (i - seg_chunk[lo]) * chunk) * 8u;
    entry[i] = reached[i] = pack_state(start, 0, 0);
    dirty[i] = 1;
  }
  __syncthreads();
  // synchronisation: decode every chunk whose entry changed up to its end, until no entry changes
  for (;;) {
    for (int i = tid; i < nch; i += nt) {
      if (!dirty[i]) continue;
      const int s = cseg[i];
      const uint32_t seg_end = (uint32_t)segs[seg0 + s + 1] * 8u;
      const uint32_t cstart = (uint32_t)(segs[seg0 + s] + (i - seg_chunk[s]) * chunk) * 8u;
      const uint32_t end = min(seg_end, cstart + (uint32_t)chunk * 8u);
      const unsigned long long e0 = entry[i];
      int4 c = make_int4(0, 0, 0, 0);
      uint32_t p = (uint32_t)e0;
      int b = (int)((e0 >> 32) & 0xff), k = (int)((e0 >> 40) & 0xff);
      while (p < end) {
        const int b0 = b;
        const uint32_t p0 = p;
        int pos, val, kend;
        bool done;
        if (jpeg_symbol(it, words, p, b, k, pos, val, kend, done) != JS_OK) {
          // a guessed entry ran into an invalid symbol: guess again one bit on, so that this chunk can still pass on
          // a state that synchronises.  An exact entry never gets here in a valid stream, and the coefficient pass
          // reports the error of an invalid one.
          p = p0 + 1;
          b = k = 0;
          continue;
        }
        if (pos == 0) {
          const int comp = b0 < it.ny ? 0 : b0 - it.ny + 1;
          if (comp == 0) c.y += val;
          else if (comp == 1) c.z += val;
          else c.w += val;
        }
        c.x += done;
      }
      const unsigned long long st = pack_state(p, b, k);
      cnt[i] = c;
      if (i + 1 < nch && cseg[i + 1] == s) reached[i + 1] = st;
    }
    __syncthreads();
    int changed = 0;
    for (int i = tid; i < nch; i += nt) {
      const bool first = seg_chunk[cseg[i]] == i;
      const bool moved = !first && reached[i] != entry[i];
      if (moved) {
        entry[i] = reached[i];
        changed = 1;
      }
      dirty[i] = moved;
    }
    if (!__syncthreads_or(changed)) break;
  }
  // blocks and DC sums before each chunk, over the image
  int4 run = make_int4(0, 0, 0, 0);
  for (int i0 = 0; i0 < nch; i0 += nt) {
    const int i = i0 + tid;
    const int4 c = i < nch ? cnt[i] : make_int4(0, 0, 0, 0);
    int4 tile, ex;
    ex.x = block_exclusive_scan(c.x, red, tile.x);
    ex.y = block_exclusive_scan(c.y, red, tile.y);
    ex.z = block_exclusive_scan(c.z, red, tile.z);
    ex.w = block_exclusive_scan(c.w, red, tile.w);
    __syncthreads();
    if (i < nch) cnt[i] = make_int4(run.x + ex.x, run.y + ex.y, run.z + ex.z, run.w + ex.w);
    run = make_int4(run.x + tile.x, run.y + tile.y, run.z + tile.z, run.w + tile.w);
  }
  __syncthreads();
  // coefficients: every chunk from its exact entry, with its block index and DC predictions
  short* out = coef + (size_t)h[JC_BLK0] * 64;
  for (int i = tid; i < nch; i += nt) {
    const int s = cseg[i], f = seg_chunk[s];
    const int4 x = cnt[i], x0 = cnt[f];
    int blk = s * ri * bpm + (x.x - x0.x);
    const int seg_end_blk = min((s + 1) * ri, total_mcus) * bpm;
    if (blk >= seg_end_blk) continue;                 // past the segment's last block: padding or trailing data
    int pred[3] = {x.y - x0.y, x.z - x0.z, x.w - x0.w};
    const uint32_t seg_end = (uint32_t)segs[seg0 + s + 1] * 8u;
    const uint32_t cstart = (uint32_t)(segs[seg0 + s] + (i - f) * chunk) * 8u;
    const bool last = i + 1 == seg_chunk[s + 1];
    const uint32_t end = last ? seg_end : min(seg_end, cstart + (uint32_t)chunk * 8u);
    const unsigned long long st = entry[i];
    int err = JS_OK;
    {
      uint32_t p = (uint32_t)st;
      int b = (int)((st >> 32) & 0xff), k = (int)((st >> 40) & 0xff);
      for (;;) {
        if (blk == seg_end_blk) {                     // this chunk ends the segment
          if (p > seg_end) err = JS_ENDS_EARLY;
          else if (seg_end - p > 7) err = JS_TRAILING;
          else atomicAdd(&s_done, 1);
          break;
        }
        if (p >= end) {
          if (last) err = JS_ENDS_EARLY;
          break;
        }
        const int k0 = k, b0 = b;
        int pos, val, kend;
        bool done;
        err = jpeg_symbol(it, words, p, b, k, pos, val, kend, done);
        if (err != JS_OK) break;
        if (p > seg_end) {
          err = JS_ENDS_EARLY;
          break;
        }
        short* blkp = out + (size_t)blk * 64;
        if (pos == 0) {
          const int comp = b0 < it.ny ? 0 : b0 - it.ny + 1;
          pred[comp] += val;
          val = pred[comp];
        }
        for (int z = k0; z < kend; ++z) blkp[kNatural[z]] = (short)(z == pos ? val : 0);
        blk += done;
      }
    }
    if (err != JS_OK) atomicMin(&s_first_err, i * 8 + err);     // the first failing chunk's error: the chunks after
                                                                 // it start from states that are not exact
  }
  __syncthreads();
  if (tid == 0) status[j] = s_first_err != INT_MAX ? (s_first_err & 7) : (s_done == nseg ? JS_OK : JS_ENDS_EARLY);
}

// jidctint.c constants (CONST_BITS 13)
constexpr int IDCT_CONST_BITS = 13, IDCT_PASS1_BITS = 2;

// jpeg_idct_islow's 1-D stage on 8 values: -> the 8 outputs before descaling (the even part from 0, 2, 4, 6, the odd
// part from 1, 3, 5, 7)
__device__ __forceinline__ void idct_1d(const int (&c)[8], int (&o)[8]) {
  int z2 = c[2], z3 = c[6];
  int z1 = (z2 + z3) * 4433;
  const int tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
  z2 = c[0];
  z3 = c[4];
  const int tmp0 = (z2 + z3) * (1 << IDCT_CONST_BITS), tmp1 = (z2 - z3) * (1 << IDCT_CONST_BITS);
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int a0 = c[7], a1 = c[5], a2 = c[3], a3 = c[1];
  z1 = a0 + a3;
  z2 = a1 + a2;
  z3 = a0 + a2;
  int z4 = a1 + a3;
  const int z5 = (z3 + z4) * 9633;
  a0 *= 2446;
  a1 *= 16819;
  a2 *= 25172;
  a3 *= 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  a0 += z1 + z3;
  a1 += z2 + z4;
  a2 += z2 + z3;
  a3 += z1 + z4;
  o[0] = t10 + a3;
  o[7] = t10 - a3;
  o[1] = t11 + a2;
  o[6] = t11 - a2;
  o[2] = t12 + a1;
  o[5] = t12 - a1;
  o[3] = t13 + a0;
  o[4] = t13 - a0;
}

__device__ __forceinline__ int idct_descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// the post-IDCT range limit: (x & 1023) through libjpeg's table is the 10-bit wrap of x, clamped, around 128
__device__ __forceinline__ unsigned char idct_limit(int x) {
  const int v = (((x + 512) & 1023) - 512) + 128;
  return (unsigned char)(v < 0 ? 0 : v > 255 ? 255 : v);
}

constexpr int IDCT_THREADS = 256, IMAGE_CTAS = 32;

__device__ __forceinline__ int plane_offset(const int* h, int comp) {
  const int mx = h[JC_MCUX], my = h[JC_MCUY];
  const int ysize = mx * h[JC_HY] * 8 * my * h[JC_VY] * 8;
  return h[JC_PLANE0] + (comp == 0 ? 0 : ysize + (comp - 1) * mx * 8 * my * 8);
}

// One thread per block of image blockIdx.y, in decode order: its place in its component's plane from the MCU layout.
__global__ void __launch_bounds__(IDCT_THREADS) jpeg_idct_kernel(const short* __restrict__ coef,
                                                                  const int* __restrict__ header,
                                                                  const int* __restrict__ qtabs,
                                                                  unsigned char* __restrict__ planes) {
  const int* h = header + (size_t)blockIdx.y * JPEG_COLS;
  const int ncomp = h[JC_NCOMP], hy = h[JC_HY], vy = h[JC_VY], mcux = h[JC_MCUX];
  const int ny = hy * vy, bpm = ny + ncomp - 1;
  const int nblk = mcux * h[JC_MCUY] * bpm;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < nblk; t += gridDim.x * blockDim.x) {
    const int m = t / bpm, b = t - m * bpm;
    const int comp = b < ny ? 0 : b - ny + 1;
    const int hc = comp ? 1 : hy, vc = comp ? 1 : vy;
    const int bv = comp ? 0 : b / hy, bh = comp ? 0 : b - (b / hy) * hy;
    const int my_ = m / mcux, mx_ = m - my_ * mcux;
    const int bx = mx_ * hc + bh, by = my_ * vc + bv;
    const int pw = mcux * hc * 8;
    const int* q = qtabs + (size_t)h[JC_Q0 + comp] * 64;
    const int4* src = (const int4*)(coef + ((size_t)h[JC_BLK0] + t) * 64);
    int d[64];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int4 v = src[r];
      const int w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        d[8 * r + 2 * e] = (int)(short)(w[e] & 0xffff) * q[8 * r + 2 * e];
        d[8 * r + 2 * e + 1] = (int)(short)(w[e] >> 16) * q[8 * r + 2 * e + 1];
      }
    }
    int ws[64];
#pragma unroll
    for (int x = 0; x < 8; ++x) {                     // pass 1: columns
      int c[8], o[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) c[u] = d[8 * u + x];
      idct_1d(c, o);
#pragma unroll
      for (int y = 0; y < 8; ++y) ws[8 * y + x] = idct_descale(o[y], IDCT_CONST_BITS - IDCT_PASS1_BITS);
    }
    unsigned char* dst = planes + plane_offset(h, comp) + (size_t)(by * 8) * pw + bx * 8;
#pragma unroll
    for (int y = 0; y < 8; ++y) {                     // pass 2: rows
      int c[8], o[8];
#pragma unroll
      for (int v = 0; v < 8; ++v) c[v] = ws[8 * y + v];
      idct_1d(c, o);
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        lo |= (uint32_t)idct_limit(idct_descale(o[x], IDCT_CONST_BITS + IDCT_PASS1_BITS + 3)) << (8 * x);
        hi |= (uint32_t)idct_limit(idct_descale(o[x + 4], IDCT_CONST_BITS + IDCT_PASS1_BITS + 3)) << (8 * x);
      }
      *(uint2*)(dst + (size_t)y * pw) = make_uint2(lo, hi);
    }
  }
}

// jdsample.c's upsampled chroma sample at output (x, y) of a component plane c (row stride pw; dw x dh real samples)
__device__ __forceinline__ int chroma_at(const unsigned char* __restrict__ c, int pw, int x, int y, int hy, int vy,
                                         int dw, int dh) {
  if (hy == 1) return c[(size_t)y * pw + x];
  const int i = x >> 1;
  if (vy == 1) {                                      // h2v1
    const unsigned char* r = c + (size_t)y * pw;
    if (dw <= 2) return r[i];
    if (!(x & 1)) return i == 0 ? r[0] : (3 * r[i] + r[i - 1] + 1) >> 2;
    return i == dw - 1 ? r[i] : (3 * r[i] + r[i + 1] + 2) >> 2;
  }
  const int row = y >> 1;                             // h2v2
  const unsigned char* n = c + (size_t)row * pw;
  if (dw <= 2) return n[i];
  const int far_row = (y & 1) ? min(row + 1, dh - 1) : max(row - 1, 0);
  const unsigned char* f = c + (size_t)far_row * pw;
  const int cs = 3 * n[i] + f[i];
  if (!(x & 1)) return i == 0 ? (cs * 4 + 8) >> 4 : (3 * cs + 3 * n[i - 1] + f[i - 1] + 8) >> 4;
  return i == dw - 1 ? (cs * 4 + 7) >> 4 : (3 * cs + 3 * n[i + 1] + f[i + 1] + 7) >> 4;
}

// One thread per output pixel of image blockIdx.y: the upsampled chroma, then jdcolor.c's ycc_rgb_convert tables
// (16-bit fixed point), or the grey value three times.
__global__ void __launch_bounds__(IDCT_THREADS) jpeg_color_kernel(const unsigned char* __restrict__ planes,
                                                                   const int* __restrict__ header,
                                                                   const long long* __restrict__ offsets,
                                                                   unsigned char* __restrict__ pixels) {
  const int* h = header + (size_t)blockIdx.y * JPEG_COLS;
  const int W = h[JC_W], H = h[JC_H], ncomp = h[JC_NCOMP], hy = h[JC_HY], vy = h[JC_VY], mcux = h[JC_MCUX];
  const unsigned char* yp = planes + plane_offset(h, 0);
  const int pw0 = mcux * hy * 8, pw1 = mcux * 8;
  const unsigned char* cbp = planes + plane_offset(h, 1);
  const unsigned char* crp = planes + plane_offset(h, 2);
  const int dw = (W + hy - 1) / hy, dh = (H + vy - 1) / vy;
  unsigned char* out = pixels + offsets[h[JC_IMG]];
  const int npix = W * H;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < npix; t += gridDim.x * blockDim.x) {
    const int y = t / W, x = t - y * W;
    const int Y = yp[(size_t)y * pw0 + x];
    int r = Y, g = Y, b = Y;
    if (ncomp == 3) {
      const int cb = chroma_at(cbp, pw1, x, y, hy, vy, dw, dh) - 128;
      const int cr = chroma_at(crp, pw1, x, y, hy, vy, dw, dh) - 128;
      r = Y + ((91881 * cr + 32768) >> 16);
      g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
      b = Y + ((116130 * cb + 32768) >> 16);
      r = r < 0 ? 0 : r > 255 ? 255 : r;
      g = g < 0 ? 0 : g > 255 ? 255 : g;
      b = b < 0 ? 0 : b > 255 ? 255 : b;
    }
    out[(size_t)t * 3] = (unsigned char)r;
    out[(size_t)t * 3 + 1] = (unsigned char)g;
    out[(size_t)t * 3 + 2] = (unsigned char)b;
  }
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_jpeg_header_cols(void) { return JPEG_COLS; }

size_t hk_jpeg_workspace_bytes(int J, int G, long long scan_bytes, int chunk_bytes) {
  if (J <= 0 || G < J || scan_bytes < 0 || chunk_bytes <= 0) return 0;
  return huff_ws_bytes(J, G, huff_chunks_bound(J, G, scan_bytes, chunk_bytes));
}

int hk_jpeg_huffman(const unsigned char* scan, const int* segs, const int* header, const unsigned char* htabs,
                    short* coef, int* status, int J, int G, long long scan_bytes, int chunk_bytes, void* workspace,
                    size_t workspace_bytes, void* stream) {
  HK_REQUIRE(scan && segs && header && htabs && coef && status && workspace, HK_ERR_ARG, "hk_jpeg_huffman: null pointer");
  HK_REQUIRE(J > 0 && G >= J && scan_bytes > 8 && scan_bytes < (1LL << 28) && chunk_bytes > 0, HK_ERR_ARG,
             "hk_jpeg_huffman: bad J=%d, G=%d, scan_bytes=%lld or chunk_bytes=%d", J, G, scan_bytes, chunk_bytes);
  HK_REQUIRE(((uintptr_t)scan & 3) == 0, HK_ERR_ALIGN, "hk_jpeg_huffman: scan must be 4-byte aligned");
  const long long nch = huff_chunks_bound(J, G, scan_bytes, chunk_bytes);
  HK_REQUIRE(workspace_bytes >= huff_ws_bytes(J, G, nch), HK_ERR_WORKSPACE, "hk_jpeg_huffman: workspace too small");
  jpeg_huffman_kernel<<<J, HUFF_THREADS, 0, (cudaStream_t)stream>>>(
      (const uint32_t*)scan, segs, header, (const HuffTab*)htabs, coef, status, chunk_bytes,
      huff_ws(workspace, J, G, nch));
  HK_LAUNCH_CHECK("jpeg_huffman_kernel");
  return 0;
}

int hk_jpeg_idct(const short* coef, const int* header, const int* qtabs, unsigned char* planes, int J, void* stream) {
  HK_REQUIRE(coef && header && qtabs && planes, HK_ERR_ARG, "hk_jpeg_idct: null pointer");
  HK_REQUIRE(J > 0 && J <= 65535, HK_ERR_ARG, "hk_jpeg_idct: bad J=%d", J);
  HK_REQUIRE(((uintptr_t)coef & 15) == 0 && ((uintptr_t)planes & 7) == 0, HK_ERR_ALIGN,
             "hk_jpeg_idct: coef must be 16-byte and planes 8-byte aligned");
  jpeg_idct_kernel<<<dim3(IMAGE_CTAS, J), IDCT_THREADS, 0, (cudaStream_t)stream>>>(coef, header, qtabs, planes);
  HK_LAUNCH_CHECK("jpeg_idct_kernel");
  return 0;
}

int hk_jpeg_color(const unsigned char* planes, const int* header, const long long* offsets, unsigned char* pixels,
                  int J, void* stream) {
  HK_REQUIRE(planes && header && offsets && pixels, HK_ERR_ARG, "hk_jpeg_color: null pointer");
  HK_REQUIRE(J > 0 && J <= 65535, HK_ERR_ARG, "hk_jpeg_color: bad J=%d", J);
  jpeg_color_kernel<<<dim3(IMAGE_CTAS, J), IDCT_THREADS, 0, (cudaStream_t)stream>>>(planes, header, offsets, pixels);
  HK_LAUNCH_CHECK("jpeg_color_kernel");
  return 0;
}

}  // extern "C"
