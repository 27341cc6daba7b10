// The default train and eval transform presets (dataset/transforms.py ClassificationPresetTrain / ClassificationPresetEval)
// on the GPU, from decoded uint8 images to the model's fp32 NCHW input:
//   * crop-resize with the arithmetic of PIL's Image.resize(BILINEAR): a separable filter whose support grows with the
//     downscale factor, 22-bit fixed-point coefficients, the horizontal pass rounded to uint8 before the vertical pass, a
//     pass whose size does not change skipped.  RandomResizedCrop, RandomHorizontalFlip and Resize + CenterCrop are all one
//     geometry: a source box resized to a virtual size, of which an S x S window is kept, optionally mirrored.
//   * the per-image table of TrivialAugmentWide's Contrast / AutoContrast / Equalize (PIL's ImageEnhance / ImageOps).
//   * TrivialAugmentWide's op (torchvision autoaugment._apply_op on a PIL image), ToTensor, Normalize and RandomErasing.
// Every random draw is made on the host, by the same torchvision calls as the host presets; the kernels read the results
// from a double table [N, AUG_COLS] (hawkeye_b200/ops_augment.py writes it).  Doubles and the _rn intrinsics keep PIL's
// double-precision steps (coefficients, affine coordinates, the LUT scales) in PIL's operation order, without contraction
// into FMAs; the blends are PIL's float steps in the same way.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

// columns of the parameter table
enum AugCol {
  AC_BX, AC_BY, AC_BW, AC_BH,   // source box (x, y, width, height), inside the image
  AC_VW, AC_VH,                 // virtual size the box is resized to
  AC_WX, AC_WY,                 // origin of the kept S x S window in the virtual image (outside it: 0, CenterCrop's pad)
  AC_FLIP,                      // 1: the window is mirrored left-right
  AC_OP, AC_MAG,                // TrivialAugmentWide op (AugOp) and its signed magnitude, as _apply_op receives them
  AC_M0,                        // 6 entries: PIL's inverse affine matrix of the geometric ops (output -> input)
  AC_EI = AC_M0 + 6, AC_EJ, AC_EH, AC_EW,   // RandomErasing rectangle (top, left, height, width); height 0: none
  AUG_COLS
};

// TrivialAugmentWide._augmentation_space order
enum AugOp {
  OP_IDENTITY, OP_SHEAR_X, OP_SHEAR_Y, OP_TRANSLATE_X, OP_TRANSLATE_Y, OP_ROTATE, OP_BRIGHTNESS, OP_COLOR, OP_CONTRAST,
  OP_SHARPNESS, OP_POSTERIZE, OP_SOLARIZE, OP_AUTOCONTRAST, OP_EQUALIZE, OP_COUNT
};

constexpr int PIL_PRECISION_BITS = 32 - 8 - 2;   // Resample.c

// Resample.c precompute_coeffs for one output index of a bilinear pass (support 1): taps [first, first + count) of the
// input, their weight sum, and what each weight needs.  in0 = 0 (the box is the whole of the cropped input).
struct PilTaps {
  int first, count;
  double center, ss, ww;
};

__device__ __forceinline__ double pil_weight(const PilTaps& t, int x) {
  double d = __dmul_rn(__dadd_rn(__dsub_rn((double)(x + t.first), t.center), 0.5), t.ss);
  d = fabs(d);
  return d < 1.0 ? __dsub_rn(1.0, d) : 0.0;
}

__device__ __forceinline__ PilTaps pil_taps(int in_size, int out_size, int o) {
  PilTaps t;
  const double scale = __ddiv_rn((double)in_size, (double)out_size);
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = fs;
  t.center = __dmul_rn(__dadd_rn((double)o, 0.5), scale);
  t.ss = __ddiv_rn(1.0, fs);
  int lo = (int)__dadd_rn(__dsub_rn(t.center, support), 0.5);
  int hi = (int)__dadd_rn(__dadd_rn(t.center, support), 0.5);
  lo = lo < 0 ? 0 : lo;
  hi = hi > in_size ? in_size : hi;
  t.first = lo;
  t.count = hi - lo;
  t.ww = 0.0;
  for (int x = 0; x < t.count; ++x) t.ww = __dadd_rn(t.ww, pil_weight(t, x));
  return t;
}

// normalize_coeffs_8bpc: the weight / sum in PRECISION_BITS fixed point (bilinear weights are never negative)
__device__ __forceinline__ int pil_coeff(const PilTaps& t, int x) {
  double w = pil_weight(t, x);
  if (t.ww != 0.0) w = __ddiv_rn(w, t.ww);
  return (int)__dadd_rn(0.5, __dmul_rn(w, (double)(1 << PIL_PRECISION_BITS)));
}

__device__ __forceinline__ int pil_clip8(int v) {
  if (v >= (1 << PIL_PRECISION_BITS << 8)) return 255;
  if (v <= 0) return 0;
  return v >> PIL_PRECISION_BITS;
}

// One thread per output pixel of one image (blockIdx.y): every channel of both passes.  Each tap's coefficient is
// recomputed where it is used (a few double operations) rather than staged: the taps per pixel are few at the sizes
// the presets produce.
__global__ void crop_resize_kernel(const unsigned char* __restrict__ src, const long long* __restrict__ offsets,
                                   const int* __restrict__ sizes, const double* __restrict__ params,
                                   unsigned char* __restrict__ out, int S) {
  const int n = blockIdx.y;
  const double* p = params + (size_t)n * AUG_COLS;
  const int bx = (int)p[AC_BX], by = (int)p[AC_BY], bw = (int)p[AC_BW], bh = (int)p[AC_BH];
  const int vw = (int)p[AC_VW], vh = (int)p[AC_VH], wx = (int)p[AC_WX], wy = (int)p[AC_WY], flip = p[AC_FLIP] != 0.0;
  const int H = sizes[2 * n], W = sizes[2 * n + 1];
  const bool valid = bw > 0 && bh > 0 && vw > 0 && vh > 0 && bx >= 0 && by >= 0 && bx + bw <= W && by + bh <= H;
  const unsigned char* img = src + offsets[n];
  const bool need_h = vw != bw, need_v = vh != bh;
  unsigned char* o = out + (size_t)n * S * S * 3;
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < S * S; pix += gridDim.x * blockDim.x) {
    const int oy = pix / S, ox = pix - oy * S;
    const int vx = wx + (flip ? S - 1 - ox : ox), vy = wy + oy;
    int res[3] = {0, 0, 0};
    if (valid && vx >= 0 && vx < vw && vy >= 0 && vy < vh) {
      PilTaps th, tv;
      if (need_h) th = pil_taps(bw, vw, vx);
      if (need_v) tv = pil_taps(bh, vh, vy);
      const int rows = need_v ? tv.count : 1;
      int acc[3] = {1 << (PIL_PRECISION_BITS - 1), 1 << (PIL_PRECISION_BITS - 1), 1 << (PIL_PRECISION_BITS - 1)};
      for (int t = 0; t < rows; ++t) {
        const int y = need_v ? tv.first + t : vy;
        const unsigned char* row = img + ((size_t)(by + y) * W + bx) * 3;
        int h[3];
        if (need_h) {
          h[0] = h[1] = h[2] = 1 << (PIL_PRECISION_BITS - 1);
          for (int u = 0; u < th.count; ++u) {
            const int k = pil_coeff(th, u);
            const unsigned char* s = row + (th.first + u) * 3;
            h[0] += s[0] * k;
            h[1] += s[1] * k;
            h[2] += s[2] * k;
          }
          for (int c = 0; c < 3; ++c) h[c] = pil_clip8(h[c]);
        } else {
          for (int c = 0; c < 3; ++c) h[c] = row[vx * 3 + c];
        }
        if (need_v) {
          const int k = pil_coeff(tv, t);
          for (int c = 0; c < 3; ++c) acc[c] += h[c] * k;
        } else {
          for (int c = 0; c < 3; ++c) res[c] = h[c];
        }
      }
      if (need_v)
        for (int c = 0; c < 3; ++c) res[c] = pil_clip8(acc[c]);
    }
    for (int c = 0; c < 3; ++c) o[(size_t)pix * 3 + c] = (unsigned char)res[c];
  }
}

// ImageEnhance's Image.blend(degenerate, image, factor) on one 8-bit value (Blend.c; alpha is a C float)
__device__ __forceinline__ int pil_blend(int deg, int v, float alpha) {
  const float t = __fadd_rn((float)deg, __fmul_rn(alpha, (float)(v - deg)));
  if (alpha >= 0.f && alpha <= 1.f) return (int)t;
  return t <= 0.f ? 0 : t >= 255.f ? 255 : (int)t;
}

// Convert.c rgb2l: ITU-R 601-2 luma in 16-bit fixed point
__device__ __forceinline__ int pil_luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

__device__ __forceinline__ float op_factor(const double* p) { return __double2float_rn(__dadd_rn(1.0, p[AC_MAG])); }

// One block per image; images whose op needs no statistics return at once.  Contrast: the mean of the luma image,
// rounded as ImageEnhance.Contrast does, and the blend toward it as a table.  AutoContrast / Equalize: ImageOps'
// tables from the per-channel 256-bin histograms (the first and last non-empty bins, and the cumulative counts).
__global__ void __launch_bounds__(1024) augment_stats_kernel(const unsigned char* __restrict__ img,
                                                             const double* __restrict__ params,
                                                             unsigned char* __restrict__ lut, int S) {
  __shared__ int hist[3][256];
  __shared__ long long red[32];
  const int n = blockIdx.x;
  const double* p = params + (size_t)n * AUG_COLS;
  const int op = (int)p[AC_OP];
  if (op != OP_CONTRAST && op != OP_AUTOCONTRAST && op != OP_EQUALIZE) return;
  const unsigned char* x = img + (size_t)n * S * S * 3;
  unsigned char* L = lut + (size_t)n * 3 * 256;
  const int npix = S * S;
  if (op == OP_CONTRAST) {
    long long s = 0;
    for (int i = threadIdx.x; i < npix; i += blockDim.x) s += pil_luma(x[3 * i], x[3 * i + 1], x[3 * i + 2]);
    s = block_sum(s, red);
    // ImageStat.Stat(L).mean = sum / count (a double), then int(mean + 0.5)
    const int mean = (int)__dadd_rn(__ddiv_rn((double)s, (double)npix), 0.5);
    const float f = op_factor(p);
    for (int i = threadIdx.x; i < 256; i += blockDim.x) L[i] = L[256 + i] = L[512 + i] = (unsigned char)pil_blend(mean, i, f);
    return;
  }
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) (&hist[0][0])[i] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < npix; i += blockDim.x)
    for (int c = 0; c < 3; ++c) atomicAdd(&hist[c][x[3 * i + c]], 1);
  __syncthreads();
  if (threadIdx.x >= 3) return;
  const int c = threadIdx.x;
  const int* h = hist[c];
  unsigned char* l = L + c * 256;
  bool identity = true;
  if (op == OP_AUTOCONTRAST) {                               // ImageOps.autocontrast(cutoff=0, ignore=None)
    int lo = 0, hi = 255;
    while (lo < 255 && !h[lo]) ++lo;
    while (hi > 0 && !h[hi]) --hi;
    if (hi > lo) {
      identity = false;
      const double scale = __ddiv_rn(255.0, (double)(hi - lo));
      const double offset = __dmul_rn((double)(-lo), scale);
      for (int i = 0; i < 256; ++i) {
        int v = (int)__dadd_rn(__dmul_rn((double)i, scale), offset);
        l[i] = (unsigned char)(v < 0 ? 0 : v > 255 ? 255 : v);
      }
    }
  } else {                                                   // ImageOps.equalize
    int nonempty = 0, total = 0, last = 0;
    for (int i = 0; i < 256; ++i)
      if (h[i]) { ++nonempty; total += h[i]; last = h[i]; }
    const int step = nonempty > 1 ? (total - last) / 255 : 0;
    if (step) {
      identity = false;
      int m = step / 2;
      for (int i = 0; i < 256; ++i) {
        const int v = m / step;
        l[i] = (unsigned char)(v > 255 ? 255 : v);           // Image.point clips its table to 8 bits
        m += h[i];
      }
    }
  }
  if (identity)
    for (int i = 0; i < 256; ++i) l[i] = (unsigned char)i;
}

// PIL's bilinear_filter32RGB (Geometry.c) at input position (xin, yin); false outside the image (the fill, 0, stays)
__device__ __forceinline__ bool pil_bilinear(const unsigned char* __restrict__ x, int S, double xin, double yin, int v[3]) {
  if (xin < 0.0 || xin >= (double)S || yin < 0.0 || yin >= (double)S) return false;
  xin = __dsub_rn(xin, 0.5);
  yin = __dsub_rn(yin, 0.5);
  const int xi = (int)floor(xin), yi = (int)floor(yin);
  const double dx = __dsub_rn(xin, (double)xi), dy = __dsub_rn(yin, (double)yi);
  const int x0 = xi < 0 ? 0 : (xi < S ? xi : S - 1), x1 = xi + 1 < 0 ? 0 : (xi + 1 < S ? xi + 1 : S - 1);
  const int y0 = yi < 0 ? 0 : (yi < S ? yi : S - 1);
  const bool has_y1 = yi + 1 >= 0 && yi + 1 < S;
  for (int c = 0; c < 3; ++c) {
    const unsigned char* r0 = x + (size_t)y0 * S * 3 + c;
    const double a0 = r0[x0 * 3], b0 = r0[x1 * 3];
    const double v1 = __dadd_rn(a0, __dmul_rn(__dsub_rn(b0, a0), dx));
    double v2 = v1;
    if (has_y1) {
      const unsigned char* r1 = x + (size_t)(yi + 1) * S * 3 + c;
      const double a1 = r1[x0 * 3], b1 = r1[x1 * 3];
      v2 = __dadd_rn(a1, __dmul_rn(__dsub_rn(b1, a1), dx));
    }
    v[c] = (int)__dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy));
  }
  return true;
}

// ImageFilter.SMOOTH (Filter.c ImagingFilter3x3: float kernel/13, rows y+1, y, y-1, offset 0.5 then truncation) at an
// interior pixel
__device__ __forceinline__ int pil_smooth(const unsigned char* __restrict__ x, int S, int y, int xx, int c) {
  const float k = 1.f / 13.f, k5 = 5.f / 13.f;
  float ss = 0.5f;
  for (int dy = 1; dy >= -1; --dy) {
    const unsigned char* r = x + ((size_t)(y + dy) * S + xx) * 3 + c;
    const float kc = dy == 0 ? k5 : k;
    ss = __fadd_rn(ss, __fadd_rn(__fadd_rn(__fmul_rn((float)r[-3], k), __fmul_rn((float)r[0], kc)), __fmul_rn((float)r[3], k)));
  }
  return ss <= 0.f ? 0 : ss >= 255.f ? 255 : (int)ss;
}

constexpr int APPLY_PIX_PER_THREAD = 8;

// One image per blockIdx.y; the image's op, then /255, Normalize and the erasing rectangle, written as fp32 NCHW.
__global__ void augment_apply_kernel(const unsigned char* __restrict__ img, const double* __restrict__ params,
                                     const unsigned char* __restrict__ lut, float* __restrict__ out, int S, float m0,
                                     float m1, float m2, float i0, float i1, float i2) {
  __shared__ unsigned char tab[3][256];
  const int n = blockIdx.y;
  const double* p = params + (size_t)n * AUG_COLS;
  const int op = (int)p[AC_OP];
  const unsigned char* x = img + (size_t)n * S * S * 3;
  const bool table = op == OP_BRIGHTNESS || op == OP_POSTERIZE || op == OP_SOLARIZE || op == OP_CONTRAST ||
                     op == OP_AUTOCONTRAST || op == OP_EQUALIZE;
  if (table) {
    const float f = op_factor(p);
    const double mag = p[AC_MAG];
    const int bits = (int)mag;
    for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) {
      const int v = i & 255;
      int r;
      if (op == OP_BRIGHTNESS) r = pil_blend(0, v, f);
      else if (op == OP_POSTERIZE) r = v & ~((1 << (8 - bits)) - 1);
      else if (op == OP_SOLARIZE) r = (double)v < mag ? v : 255 - v;
      else r = lut[(size_t)n * 3 * 256 + i];
      (&tab[0][0])[i] = (unsigned char)r;
    }
    __syncthreads();
  }
  const bool geometric = op >= OP_SHEAR_X && op <= OP_ROTATE;
  const double a0 = p[AC_M0], a1 = p[AC_M0 + 1], a2 = p[AC_M0 + 2], a3 = p[AC_M0 + 3], a4 = p[AC_M0 + 4],
               a5 = p[AC_M0 + 5];
  const float f = op_factor(p);
  const int ei = (int)p[AC_EI], ej = (int)p[AC_EJ], eh = (int)p[AC_EH], ew = (int)p[AC_EW];
  const size_t hw = (size_t)S * S;
  float* o = out + (size_t)n * 3 * hw;
  const int npix = S * S;
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += gridDim.x * blockDim.x) {
    const int y = pix / S, xx = pix - y * S;
    const unsigned char* s = x + (size_t)pix * 3;
    int v[3] = {s[0], s[1], s[2]};
    if (geometric) {
      // Geometry.c affine_transform at the pixel centre
      const double xc = (double)xx + 0.5, yc = (double)y + 0.5;
      const double xin = __dadd_rn(__dadd_rn(__dmul_rn(a0, xc), __dmul_rn(a1, yc)), a2);
      const double yin = __dadd_rn(__dadd_rn(__dmul_rn(a3, xc), __dmul_rn(a4, yc)), a5);
      if (!pil_bilinear(x, S, xin, yin, v)) v[0] = v[1] = v[2] = 0;
    } else if (op == OP_COLOR) {
      const int l = pil_luma(v[0], v[1], v[2]);
      for (int c = 0; c < 3; ++c) v[c] = pil_blend(l, v[c], f);
    } else if (op == OP_SHARPNESS) {
      if (y > 0 && y < S - 1 && xx > 0 && xx < S - 1)        // the border keeps the image's own pixels
        for (int c = 0; c < 3; ++c) v[c] = pil_blend(pil_smooth(x, S, y, xx, c), v[c], f);
    } else if (table) {
      for (int c = 0; c < 3; ++c) v[c] = tab[c][v[c]];
    }
    const bool erased = y >= ei && y < ei + eh && xx >= ej && xx < ej + ew;
    o[pix] = erased ? 0.f : normalize_u8_value((unsigned char)v[0], m0, i0);
    o[hw + pix] = erased ? 0.f : normalize_u8_value((unsigned char)v[1], m1, i1);
    o[2 * hw + pix] = erased ? 0.f : normalize_u8_value((unsigned char)v[2], m2, i2);
  }
}

// blocks per image of a kernel over S*S pixels: 256-thread blocks, about APPLY_PIX_PER_THREAD pixels per thread
inline int blocks_per_image(int S) {
  const int per_block = 256 * APPLY_PIX_PER_THREAD;
  const int b = (int)(((size_t)S * S + per_block - 1) / per_block);
  return b < 1 ? 1 : b;
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_augment_params_cols(void) { return AUG_COLS; }

int hk_augment_crop_resize(const unsigned char* src, const long long* offsets, const int* sizes, const double* params,
                           unsigned char* out, int N, int S, void* stream) {
  HK_REQUIRE(src && offsets && sizes && params && out, HK_ERR_ARG, "hk_augment_crop_resize: null pointer");
  HK_REQUIRE(N > 0 && N <= 65535 && S > 0 && S <= 8192, HK_ERR_ARG, "hk_augment_crop_resize: bad N=%d or S=%d", N, S);
  crop_resize_kernel<<<dim3(blocks_per_image(S), N), 256, 0, (cudaStream_t)stream>>>(src, offsets, sizes, params, out, S);
  HK_LAUNCH_CHECK("crop_resize_kernel");
  return 0;
}

int hk_augment_stats(const unsigned char* img, const double* params, unsigned char* lut, int N, int S, void* stream) {
  HK_REQUIRE(img && params && lut, HK_ERR_ARG, "hk_augment_stats: null pointer");
  HK_REQUIRE(N > 0 && S > 0 && S <= 8192, HK_ERR_ARG, "hk_augment_stats: bad N=%d or S=%d", N, S);
  augment_stats_kernel<<<N, 1024, 0, (cudaStream_t)stream>>>(img, params, lut, S);
  HK_LAUNCH_CHECK("augment_stats_kernel");
  return 0;
}

int hk_augment_apply(const unsigned char* img, const double* params, const unsigned char* lut, float* out, int N, int S,
                     float mean0, float mean1, float mean2, float std0, float std1, float std2, void* stream) {
  HK_REQUIRE(img && params && lut && out, HK_ERR_ARG, "hk_augment_apply: null pointer");
  HK_REQUIRE(N > 0 && N <= 65535 && S > 0 && S <= 8192, HK_ERR_ARG, "hk_augment_apply: bad N=%d or S=%d", N, S);
  HK_REQUIRE(std0 > 0.f && std1 > 0.f && std2 > 0.f, HK_ERR_ARG, "hk_augment_apply: std must be positive");
  augment_apply_kernel<<<dim3(blocks_per_image(S), N), 256, 0, (cudaStream_t)stream>>>(
      img, params, lut, out, S, mean0, mean1, mean2, 1.f / std0, 1.f / std1, 1.f / std2);
  HK_LAUNCH_CHECK("augment_apply_kernel");
  return 0;
}

}  // extern "C"
