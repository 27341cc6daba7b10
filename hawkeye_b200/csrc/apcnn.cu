// AP-CNN (reference model/methods/APCNN.py): the top-down lateral add of the feature pyramid, the pyramid attention (spatial
// gate and the two pooled vectors the heads consume, so the attended maps A3..A5 are never written), the ROI selection of
// the three levels, the ROI-guided refinement of the layer2 map with its gather-form backward, and the small vector ops of
// the heads.  The reference loops over the images on the host for the NMS (:444-476) and the crops (:478-531); nothing here
// leaves the device.  Every sum runs in a fixed order (no atomics): the same bits on every run.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

constexpr int AP_C = 256;           // channels of the pyramid maps (PyramidFeatures feature_size, :205)
constexpr int AP_CHUNK = 64;        // pixels of one image a block of the attention passes covers
constexpr int AP_DW = 9 * AP_C;     // gate weights
constexpr int AP_ROW = AP_DW + 16;  // one block's share of (dw, db), 16-byte aligned rows
constexpr int AP_ROIS = 9;

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 fma4(float s, float4 a, float4 b) {
  return make_float4(fmaf(s, a.x, b.x), fmaf(s, a.y, b.y), fmaf(s, a.z, b.z), fmaf(s, a.w, b.w));
}

// ---------------------------------------------------------------------------------------------------------------
// feature pyramid: out = up2_nearest(top) + lat, its adjoint (the 2x2 sum), a per-image row broadcast and the NHWC pool
// ---------------------------------------------------------------------------------------------------------------
__global__ void ap_lateral_fwd_kernel(const float* __restrict__ top, const float* __restrict__ lat, float* __restrict__ out,
                                      int N, int h, int w, int C4) {
  const size_t total = (size_t)N * 4 * h * w * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    size_t p = i / C4;
    const int x = (int)(p % (2 * w));
    p /= 2 * w;
    const int y = (int)(p % (2 * h)), n = (int)(p / (2 * h));
    const float4 a = ld4(top + (((size_t)n * h + (y >> 1)) * w + (x >> 1)) * C4 * 4 + c * 4), b = ld4(lat + i * 4);
    st4(out + i * 4, make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w));
  }
}

__global__ void ap_lateral_bwd_kernel(const float* __restrict__ dout, float* __restrict__ dtop, int N, int h, int w, int C4) {
  const size_t total = (size_t)N * h * w * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    size_t p = i / C4;
    const int x = (int)(p % w);
    p /= w;
    const int y = (int)(p % h), n = (int)(p / h);
    const float* r0 = dout + (((size_t)n * 2 * h + 2 * y) * 2 * w + 2 * x) * C4 * 4 + c * 4;
    const float* r1 = r0 + (size_t)2 * w * C4 * 4;
    const float4 a = ld4(r0), b = ld4(r0 + C4 * 4), d = ld4(r1), e = ld4(r1 + C4 * 4);
    st4(dtop + i * 4, make_float4((a.x + b.x) + (d.x + e.x), (a.y + b.y) + (d.y + e.y), (a.z + b.z) + (d.z + e.z),
                                  (a.w + b.w) + (d.w + e.w)));
  }
}

// y[n, p, c] = a[n, p, c] (0 without a) + scale b[n, c]
__global__ void ap_bcast_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ y, int N, int HW,
                                int C4, float scale) {
  const size_t total = (size_t)N * HW * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4), n = (int)(i / ((size_t)HW * C4));
    const float4 v = ld4(b + ((size_t)n * C4 + c) * 4);
    const float4 u = a ? ld4(a + i * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    st4(y + i * 4, fma4(scale, v, u));
  }
}

// Spatial sums of an NHWC map in two fixed-order steps: a block adds `chunk` pixels of one image for 256 channels (four
// pixel rows in flight, combined in ascending order), then one thread per (n, c) adds the blocks' shares in ascending order.
// With a gate s [N, HW] the block also adds s F (the attended pool).
template <bool GATE>
__global__ void ap_pool_partial_kernel(const float* __restrict__ x, const float* __restrict__ gate, float* __restrict__ part,
                                       int HW, int C, int chunk, int chunks) {
  __shared__ float4 red[2][4][64];
  const int n = blockIdx.y, ck = blockIdx.x, c4 = blockIdx.z * 64 + (threadIdx.x & 63), r = threadIdx.x >> 6;
  const int p0 = ck * chunk, p1 = min(HW, p0 + chunk);
  float4 af = make_float4(0.f, 0.f, 0.f, 0.f), as = af;
  for (int p = p0 + r; p < p1; p += 4) {
    const float4 f = ld4(x + ((size_t)n * HW + p) * C + c4 * 4);
    af = make_float4(af.x + f.x, af.y + f.y, af.z + f.z, af.w + f.w);
    if (GATE) as = fma4(gate[(size_t)n * HW + p], f, as);
  }
  red[0][r][threadIdx.x & 63] = af;
  if (GATE) red[1][r][threadIdx.x & 63] = as;
  __syncthreads();
  if (r == 0) {
    for (int k = 0; k < (GATE ? 2 : 1); ++k) {
      float4 t = red[k][0][threadIdx.x];
      for (int j = 1; j < 4; ++j) {
        const float4 u = red[k][j][threadIdx.x];
        t = make_float4(t.x + u.x, t.y + u.y, t.z + u.z, t.w + u.w);
      }
      st4(part + ((((size_t)n * chunks + ck) * (GATE ? 2 : 1) + k) * C) + c4 * 4, t);
    }
  }
}

// out_k[n, c] = scale * sum over the chunks of part[n, chunk, k, c], k < K
__global__ void ap_pool_final_kernel(const float* __restrict__ part, float* __restrict__ out0, float* __restrict__ out1, int N,
                                     int C, int chunks, int K, float scale) {
  const int total = N * K * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i % C, k = (i / C) % K, n = i / (C * K);
    float s = 0.f;
    for (int j = 0; j < chunks; ++j) s += part[(((size_t)n * chunks + j) * K + k) * C + c];
    (k == 0 ? out0 : out1)[(size_t)n * C + c] = s * scale;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// pyramid attention.  SpatialGate is ConvTranspose2d(256, 1, 3, 1, 1) (:276): out[y, x] = b + sum_{ky, kx}
// <F[y + 1 - ky, x + 1 - kx, :], w[:, 0, ky, kx]>.  Pass one reads F once and leaves the nine per-pixel products
// t[p, k] = <F[p, :], w[:, k]>; the gate of a pixel is then the sum of t[p + (1 - ky, 1 - kx), k] over its neighbours.
// ---------------------------------------------------------------------------------------------------------------
// Eight lanes per pixel (32 channels each, as 8 float4 128 bytes apart), four pixels per lane group in flight so that a
// weight read from shared memory serves four pixels: a warp covers 16 pixels per step.
__global__ void ap_att_taps_kernel(const float* __restrict__ F, const float* __restrict__ w, float* __restrict__ T, size_t P) {
  __shared__ __align__(16) float wT[9][AP_C];
  for (int i = threadIdx.x; i < AP_DW; i += blockDim.x) wT[i % 9][i / 9] = w[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, g = lane >> 3, l8 = lane & 7;
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t base = ((size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 16; base < P; base += nwarps * 16) {
    float acc[4][9];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int k = 0; k < 9; ++k) acc[i][k] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = 4 * (l8 + 8 * j);
      float4 f[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const size_t p = base + g * 4 + i;
        f[i] = p < P ? ld4(F + p * AP_C + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const float4 wv = ld4(&wT[k][c]);
#pragma unroll
        for (int i = 0; i < 4; ++i)
          acc[i][k] = fmaf(f[i].w, wv.w, fmaf(f[i].z, wv.z, fmaf(f[i].y, wv.y, fmaf(f[i].x, wv.x, acc[i][k]))));
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        float v = acc[i][k];
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        const size_t p = base + g * 4 + i;
        if (p < P && (l8 == k || (l8 == 0 && k == 8))) T[p * 9 + k] = v;
      }
  }
}

// One block per (chunk of 64 pixels, image): the gates of the chunk from the tap products (written to `gate`), then the
// chunk's shares of sum F and sum s F.
__global__ void ap_att_pool_kernel(const float* __restrict__ F, const float* __restrict__ T, const float* __restrict__ bias,
                                   float* __restrict__ gate, float* __restrict__ part, int H, int W, int chunks) {
  __shared__ float s_sm[AP_CHUNK];
  __shared__ float4 red[2][4][64];
  const int n = blockIdx.y, ck = blockIdx.x, HW = H * W;
  if (threadIdx.x < AP_CHUNK) {
    const int p = ck * AP_CHUNK + threadIdx.x;
    if (p < HW) {
      const int y = p / W, x = p - y * W;
      float z = bias[0];
      for (int k = 0; k < 9; ++k) {
        const int yy = y + 1 - k / 3, xx = x + 1 - k % 3;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) z += T[((size_t)n * HW + yy * W + xx) * 9 + k];
      }
      const float s = 1.f / (1.f + expf(-z));
      gate[(size_t)n * HW + p] = s;
      s_sm[threadIdx.x] = s;
    }
  }
  __syncthreads();
  const int c4 = threadIdx.x & 63, r = threadIdx.x >> 6;
  float4 af = make_float4(0.f, 0.f, 0.f, 0.f), as = af;
  for (int i = r; i < AP_CHUNK && ck * AP_CHUNK + i < HW; i += 4) {
    const float4 f = ld4(F + ((size_t)n * HW + ck * AP_CHUNK + i) * AP_C + c4 * 4);
    af = make_float4(af.x + f.x, af.y + f.y, af.z + f.z, af.w + f.w);
    as = fma4(s_sm[i], f, as);
  }
  red[0][r][c4] = af;
  red[1][r][c4] = as;
  __syncthreads();
  if (r == 0)
    for (int k = 0; k < 2; ++k) {
      float4 t = red[k][0][c4];
      for (int j = 1; j < 4; ++j) {
        const float4 u = red[k][j][c4];
        t = make_float4(t.x + u.x, t.y + u.y, t.z + u.z, t.w + u.w);
      }
      st4(part + (((size_t)n * chunks + ck) * 2 + k) * AP_C + c4 * 4, t);
    }
}

// dz[p] = s (1 - s) <F[p, :], dpool_sf[n, :]> / HW: the gradient at the gate's pre-activation.  Eight lanes per pixel.
__global__ void ap_att_dz_kernel(const float* __restrict__ F, const float* __restrict__ gate, const float* __restrict__ dsf,
                                 float* __restrict__ dz, size_t P, int HW) {
  const int lane = threadIdx.x & 31, g = lane >> 3, l8 = lane & 7;
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  const float inv = 1.f / (float)HW;
  for (size_t base = ((size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 4; base < P; base += nwarps * 4) {
    const size_t p = base + g;
    float v = 0.f;
    if (p < P) {
      const float* d = dsf + (p / HW) * AP_C;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 4 * (l8 + 8 * j);
        const float4 f = ld4(F + p * AP_C + c), u = ld4(d + c);
        v = fmaf(f.w, u.w, fmaf(f.z, u.z, fmaf(f.y, u.y, fmaf(f.x, u.x, v))));
      }
    }
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    if (p < P && l8 == 0) {
      const float s = gate[p];
      dz[p] = v * inv * s * (1.f - s);
    }
  }
}

// One block per (chunk, image).  e[q, k] = dz[q + (k / 3 - 1, k % 3 - 1)] is both what w[:, k] is multiplied by in dF[q] and
// what F[q] is multiplied by in dw[:, k].  dF = dpool_f / HW + s dpool_sf / HW + sum_k e_k w_k; the block's share of
// (dw, db) goes to `part`.
__global__ void __launch_bounds__(256) ap_att_bwd_kernel(const float* __restrict__ F, const float* __restrict__ w,
                                                         const float* __restrict__ gate, const float* __restrict__ dz,
                                                         const float* __restrict__ dpf, const float* __restrict__ dsf,
                                                         float* __restrict__ dF, float* __restrict__ part, int H, int W,
                                                         int chunks) {
  __shared__ float e_sm[AP_CHUNK][9];
  __shared__ float s_sm[AP_CHUNK];
  __shared__ float z_sm[AP_CHUNK];
  __shared__ __align__(16) float red[4][9][AP_C];
  const int n = blockIdx.y, ck = blockIdx.x, HW = H * W;
  if (threadIdx.x < AP_CHUNK) {
    const int p = ck * AP_CHUNK + threadIdx.x;
    float s = 0.f, z = 0.f;
    if (p < HW) {
      const int y = p / W, x = p - y * W;
      for (int k = 0; k < 9; ++k) {
        const int yy = y - 1 + k / 3, xx = x - 1 + k % 3;
        e_sm[threadIdx.x][k] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? dz[(size_t)n * HW + yy * W + xx] : 0.f;
      }
      s = gate[(size_t)n * HW + p];
      z = dz[(size_t)n * HW + p];
    }
    s_sm[threadIdx.x] = s;
    z_sm[threadIdx.x] = z;
  }
  __syncthreads();
  const int c4 = threadIdx.x & 63, r = threadIdx.x >> 6;
  const float inv = 1.f / (float)HW;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
  if (dpf) a = ld4(dpf + (size_t)n * AP_C + c4 * 4);
  b = ld4(dsf + (size_t)n * AP_C + c4 * 4);
  a = make_float4(a.x * inv, a.y * inv, a.z * inv, a.w * inv);
  b = make_float4(b.x * inv, b.y * inv, b.z * inv, b.w * inv);
  float4 wv[9], dw[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    wv[k] = make_float4(w[(c4 * 4 + 0) * 9 + k], w[(c4 * 4 + 1) * 9 + k], w[(c4 * 4 + 2) * 9 + k], w[(c4 * 4 + 3) * 9 + k]);
    dw[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int i = r; i < AP_CHUNK && ck * AP_CHUNK + i < HW; i += 4) {
    const size_t o = ((size_t)n * HW + ck * AP_CHUNK + i) * AP_C + c4 * 4;
    const float4 f = ld4(F + o);
    float4 g = fma4(s_sm[i], b, a);
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const float e = e_sm[i][k];
      g = fma4(e, wv[k], g);
      dw[k] = fma4(e, f, dw[k]);
    }
    st4(dF + o, g);
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) st4(&red[r][k][c4 * 4], dw[k]);
  __syncthreads();
  float* row = part + ((size_t)n * chunks + ck) * AP_ROW;
  for (int i = threadIdx.x; i < AP_DW; i += blockDim.x) {
    const int k = i / AP_C, c = i - k * AP_C;
    row[i] = (red[0][k][c] + red[1][k][c]) + (red[2][k][c] + red[3][k][c]);
  }
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < AP_CHUNK; ++i) s += z_sm[i];
    row[AP_DW] = s;
  }
}

// dw [256, 1, 3, 3] and db [1] from the blocks' shares, in ascending block order
__global__ void ap_att_bwd_final_kernel(const float* __restrict__ part, float* __restrict__ dw, float* __restrict__ db, int rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > AP_DW) return;
  float s = 0.f;
  for (int j = 0; j < rows; ++j) s += part[(size_t)j * AP_ROW + i];
  if (i == AP_DW) db[0] = s;
  else dw[(i % AP_C) * 9 + i / AP_C] = s;
}

// ---------------------------------------------------------------------------------------------------------------
// ROI selection (get_att_roi, :444-476): one block per (image, level)
// ---------------------------------------------------------------------------------------------------------------
struct RoiArgs {
  const float* g[3];
  int win[3][4];          // y0, y1, x0, x1 of the central window of each level
};

__global__ void ap_roi_kernel(RoiArgs a, const unsigned char* __restrict__ keep, float* __restrict__ boxes,
                              int* __restrict__ counts, int H3, int W3, int img_h, int img_w) {
  extern __shared__ unsigned char sm_raw[];
  __shared__ double red[32];
  __shared__ float red_v[32];
  __shared__ int red_i[32];
  __shared__ int s_pick;
  const int n = blockIdx.x, lv = blockIdx.y, h = H3 >> lv, w = W3 >> lv, hw = h * w;
  const int stride = 8 << lv, half = 32 << lv, T = lv == 0 ? 5 : (lv == 1 ? 3 : 1), off = lv == 0 ? 0 : (lv == 1 ? 5 : 8);
  float* sc = reinterpret_cast<float*>(sm_raw);
  unsigned char* alive = sm_raw + (size_t)hw * sizeof(float);
  const float* g = a.g[lv] + (size_t)n * hw;
  double part = 0.0;
  for (int i = threadIdx.x; i < hw; i += blockDim.x) {
    const int y = i / w, x = i - y * w;
    const bool in = y >= a.win[lv][0] && y < a.win[lv][1] && x >= a.win[lv][2] && x < a.win[lv][3];
    const float v = in ? g[i] : 0.f;
    sc[i] = v;
    part += (double)v;
  }
  const float mean = (float)(block_sum(part, red) / (double)hw);
  for (int i = threadIdx.x; i < hw; i += blockDim.x) alive[i] = sc[i] > mean ? 1 : 0;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float* out = boxes + ((size_t)n * AP_ROIS + off) * 4;
  int cnt = 0;
  for (int t = 0; t < T; ++t) {
    // the highest score among the alive cells; equal scores go to the highest flat index, which is what the reference's
    // ascending argsort gives when it is stable (it takes the last entry of the order)
    float best = -INFINITY;
    int bi = -1;
    for (int i = threadIdx.x; i < hw; i += blockDim.x)
      if (alive[i] && sc[i] >= best) { best = sc[i]; bi = i; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi >= 0 && (bi < 0 || ob > best || (ob == best && oi > bi))) { best = ob; bi = oi; }
    }
    if (lane == 0) { red_v[warp] = best; red_i[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float v = red_v[0];
      int b = red_i[0];
      for (int k = 1; k < nw; ++k)
        if (red_i[k] >= 0 && (b < 0 || red_v[k] > v || (red_v[k] == v && red_i[k] > b))) { v = red_v[k]; b = red_i[k]; }
      s_pick = b;
      float x1 = 0.f, y1 = 0.f, x2 = 0.f, y2 = 0.f;
      if (b >= 0) {
        const int py = b / w, px = b - py * w;
        x1 = fmaxf((float)(px * stride - half), 0.f);
        y1 = fmaxf((float)(py * stride - half), 0.f);
        x2 = fminf((float)(px * stride + half), (float)(img_w - 1));
        y2 = fminf((float)(py * stride + half), (float)(img_h - 1));
      }
      out[t * 4 + 0] = x1; out[t * 4 + 1] = y1; out[t * 4 + 2] = x2; out[t * 4 + 3] = y2;
    }
    __syncthreads();
    const int pick = s_pick;
    if (pick >= 0) {
      ++cnt;
      const int py = pick / w, px = pick - py * w;
      for (int i = threadIdx.x; i < hw; i += blockDim.x) {
        if (!alive[i]) continue;
        const int dy = i / w - py, dx = i % w - px;
        if (i == pick || (dy > -8 && dy < 8 && dx > -8 && dx < 8 && !keep[(lv * 15 + dy + 7) * 15 + dx + 7])) alive[i] = 0;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[n * 3 + lv] = cnt;
}

// ---------------------------------------------------------------------------------------------------------------
// ROI-guided refinement (get_roi_crop_feat, :478-531)
// ---------------------------------------------------------------------------------------------------------------
// meta[n] = {X1, Y1, X2, Y2 of the crop window, X1, Y1, X2, Y2 of the dropped block (empty: zeros), bits of the rescale}
constexpr int AP_META = 12;

__global__ void ap_refine_meta_kernel(const float* __restrict__ boxes, const int* __restrict__ counts,
                                      const float* __restrict__ draws, int* __restrict__ meta, int N, int H, int W) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float xx1 = INFINITY, yy1 = INFINITY, xx2 = -INFINITY, yy2 = -INFINITY;
  int total = 0;
  for (int lv = 0; lv < 3; ++lv) {
    const int off = lv == 0 ? 0 : (lv == 1 ? 5 : 8);
    for (int t = 0; t < counts[n * 3 + lv]; ++t) {
      const float* b = boxes + ((size_t)n * AP_ROIS + off + t) * 4;
      xx1 = fminf(xx1, b[0] / 8.f); yy1 = fminf(yy1, b[1] / 8.f);
      xx2 = fmaxf(xx2, b[2] / 8.f); yy2 = fmaxf(yy2, b[3] / 8.f);
      ++total;
    }
  }
  int* m = meta + (size_t)n * AP_META;
  if (total == 0) { xx1 = 0.f; yy1 = 0.f; xx2 = (float)W; yy2 = (float)H; }     // no ROI at any level: the whole map
  const int X1 = (int)xx1, Y1 = (int)yy1, X2 = min((int)xx2, W), Y2 = min((int)yy2, H);
  int D[4] = {0, 0, 0, 0};
  float rate = 1.f;
  if (draws) {
    const double u = (double)draws[n * 2];
    const int lv = u < 0.3 ? 0 : (u < 0.6 ? 1 : -1);
    if (lv >= 0 && counts[n * 3 + lv] > 0) {
      const int c = counts[n * 3 + lv];
      const int t = min((int)(draws[n * 2 + 1] * (float)c), c - 1);
      const float* b = boxes + ((size_t)n * AP_ROIS + (lv == 0 ? 0 : 5) + t) * 4;
      D[0] = (int)(b[0] / 8.f); D[1] = (int)(b[1] / 8.f); D[2] = (int)(b[2] / 8.f); D[3] = (int)(b[3] / 8.f);
    }
    const int ow = max(0, min(X2, D[2]) - max(X1, D[0])), oh = max(0, min(Y2, D[3]) - max(Y1, D[1]));
    rate = ((yy2 - yy1) * (xx2 - xx1)) / (float)((Y2 - Y1) * (X2 - X1) - ow * oh);
  }
  m[0] = X1; m[1] = Y1; m[2] = X2; m[3] = Y2;
  m[4] = D[0]; m[5] = D[1]; m[6] = D[2]; m[7] = D[3];
  m[8] = __float_as_int(rate);
}

// ATen's upsample_bilinear2d source index with align_corners=False: src = in / out (o + 0.5) - 0.5 clamped at 0
__device__ __forceinline__ void ap_src(int o, int in, int out, int& i0, int& ip, float& l0, float& l1) {
  float s = ((float)in / (float)out) * ((float)o + 0.5f) - 0.5f;
  s = s < 0.f ? 0.f : s;
  i0 = (int)s;
  ip = i0 < in - 1 ? 1 : 0;
  l1 = s - (float)i0;
  l0 = 1.f - l1;
}

__global__ void ap_refine_fwd_kernel(const float* __restrict__ x, const int* __restrict__ meta, float* __restrict__ y, int N,
                                     int H, int W, int C4) {
  const size_t total = (size_t)N * H * W * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    size_t p = i / C4;
    const int ox = (int)(p % W);
    p /= W;
    const int oy = (int)(p % H), n = (int)(p / H);
    const int* m = meta + (size_t)n * AP_META;
    const float rate = __int_as_float(m[8]);
    int h0, hp, w0, wp;
    float hl0, hl1, wl0, wl1;
    ap_src(oy, m[3] - m[1], H, h0, hp, hl0, hl1);
    ap_src(ox, m[2] - m[0], W, w0, wp, wl0, wl1);
    float4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = m[1] + h0 + (k >> 1) * hp, xx = m[0] + w0 + (k & 1) * wp;
      const bool dropped = yy >= m[5] && yy < m[7] && xx >= m[4] && xx < m[6];
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      if (!dropped) {
        t = ld4(x + ((((size_t)n * H + yy) * W + xx) * C4 + c) * 4);
        t = make_float4(t.x * rate, t.y * rate, t.z * rate, t.w * rate);
      }
      v[k] = t;
    }
    float4 o;
    o.x = hl0 * (wl0 * v[0].x + wl1 * v[1].x) + hl1 * (wl0 * v[2].x + wl1 * v[3].x);
    o.y = hl0 * (wl0 * v[0].y + wl1 * v[1].y) + hl1 * (wl0 * v[2].y + wl1 * v[3].y);
    o.z = hl0 * (wl0 * v[0].z + wl1 * v[1].z) + hl1 * (wl0 * v[2].z + wl1 * v[3].z);
    o.w = hl0 * (wl0 * v[0].w + wl1 * v[1].w) + hl1 * (wl0 * v[2].w + wl1 * v[3].w);
    st4(y + i * 4, o);
  }
}

// weight of input index `i` (relative to the window) in output `o`, with the forward's arithmetic
__device__ __forceinline__ float ap_weight(int o, int i, int in, int out) {
  int i0, ip;
  float l0, l1;
  ap_src(o, in, out, i0, ip, l0, l1);
  return (i0 == i ? l0 : 0.f) + (i0 + ip == i ? l1 : 0.f);
}

// the outputs that can read input index i: src in (i - 1, i + 1), widened by one on each side against rounding
__device__ __forceinline__ void ap_range(int i, int in, int out, int& lo, int& hi) {
  const float r = (float)out / (float)in;
  lo = max(0, (int)floorf(((float)i - 0.5f) * r - 0.5f) - 1);
  hi = min(out - 1, (int)ceilf(((float)i + 1.5f) * r - 0.5f) + 1);
}

// Gather form: one thread owns four channels of one x2 element and adds, in ascending (oy, ox), the outputs that read it.
__global__ void ap_refine_bwd_kernel(const float* __restrict__ dy, const int* __restrict__ meta, float* __restrict__ dx, int N,
                                     int H, int W, int C4) {
  const size_t total = (size_t)N * H * W * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    size_t p = i / C4;
    const int xx = (int)(p % W);
    p /= W;
    const int yy = (int)(p % H), n = (int)(p / H);
    const int* m = meta + (size_t)n * AP_META;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const bool inside = yy >= m[1] && yy < m[3] && xx >= m[0] && xx < m[2];
    const bool dropped = yy >= m[5] && yy < m[7] && xx >= m[4] && xx < m[6];
    if (inside && !dropped) {
      const int ih = m[3] - m[1], iw = m[2] - m[0], hi = yy - m[1], wi = xx - m[0];
      int oy0, oy1, ox0, ox1;
      ap_range(hi, ih, H, oy0, oy1);
      ap_range(wi, iw, W, ox0, ox1);
      for (int oy = oy0; oy <= oy1; ++oy) {
        const float wy = ap_weight(oy, hi, ih, H);
        if (wy == 0.f) continue;
        for (int ox = ox0; ox <= ox1; ++ox) {
          const float wx = ap_weight(ox, wi, iw, W);
          if (wx == 0.f) continue;
          acc = fma4(wy * wx, ld4(dy + ((((size_t)n * H + oy) * W + ox) * C4 + c) * 4), acc);
        }
      }
      const float rate = __int_as_float(m[8]);
      acc = make_float4(acc.x * rate, acc.y * rate, acc.z * rate, acc.w * rate);
    }
    st4(dx + i * 4, acc);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// heads: the bottom-up channel attention with the attended pool, and mask_cat
// ---------------------------------------------------------------------------------------------------------------
// z, pm, psf, v, ch: [3, N, C] (levels 3, 4, 5).  ch_3 = sig(z_3), ch_4 = (sig(z_4) + ch_3) / 2, ch_5 = (sig(z_5) + ch_4) / 2
// (PyramidAttentions.forward, :251-268); v_l = psf_l + ch_l pm_l = mean_hw((s_l + ch_l) F_l).
__global__ void ap_mix_fwd_kernel(const float* __restrict__ z, const float* __restrict__ pm, const float* __restrict__ psf,
                                  float* __restrict__ v, float* __restrict__ ch, int NC) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < NC; i += gridDim.x * blockDim.x) {
    float c = 0.f;
    for (int l = 0; l < 3; ++l) {
      const float s = 1.f / (1.f + expf(-z[l * NC + i]));
      c = l == 0 ? s : (s + c) / 2.f;
      ch[l * NC + i] = c;
      v[l * NC + i] = fmaf(c, pm[l * NC + i], psf[l * NC + i]);
    }
  }
}

__global__ void ap_mix_bwd_kernel(const float* __restrict__ z, const float* __restrict__ pm, const float* __restrict__ ch,
                                  const float* __restrict__ dv, float* __restrict__ dz, float* __restrict__ dpm, int NC) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < NC; i += gridDim.x * blockDim.x) {
    float carry = 0.f;
    for (int l = 2; l >= 0; --l) {
      const float g = dv[l * NC + i];
      dpm[l * NC + i] = g * ch[l * NC + i];
      const float dc = fmaf(g, pm[l * NC + i], carry);
      const float ds = l == 0 ? dc : dc / 2.f;
      carry = l == 0 ? 0.f : dc / 2.f;
      const float s = 1.f / (1.f + expf(-z[l * NC + i]));
      dz[l * NC + i] = ds * s * (1.f - s);
    }
  }
}

__global__ void ap_mask_cat_kernel(const float* __restrict__ g3, const float* __restrict__ g4, const float* __restrict__ g5,
                                   float* __restrict__ out, int N, int H, int W) {
  const size_t total = (size_t)N * 3 * H * W;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)((i / W) % H), l = (int)((i / ((size_t)W * H)) % 3), n = (int)(i / ((size_t)3 * W * H));
    const float* g = l == 0 ? g3 : (l == 1 ? g4 : g5);
    const int h = H >> l, w = W >> l;
    out[i] = g[((size_t)n * h + (y >> l)) * w + (x >> l)];
  }
}

static int pool_chunk(int HW) {
  const int c = (HW + 127) / 128;
  return c < 64 ? 64 : (c + 3) / 4 * 4;
}

static size_t att_chunks(int H, int W) { return ((size_t)H * W + AP_CHUNK - 1) / AP_CHUNK; }

}  // namespace hk

using namespace hk;

extern "C" {

int hk_apcnn_lateral_fwd(const float* top, const float* lat, float* out, int N, int h, int w, int C, void* stream) {
  HK_REQUIRE(top && lat && out, HK_ERR_ARG, "hk_apcnn_lateral_fwd: null pointer");
  HK_REQUIRE(N > 0 && h > 0 && w > 0 && C > 0 && C % 4 == 0, HK_ERR_ARG, "hk_apcnn_lateral_fwd: N=%d h=%d w=%d C=%d (C %% 4)", N,
             h, w, C);
  HK_REQUIRE(aligned16(top) && aligned16(lat) && aligned16(out), HK_ERR_ALIGN, "hk_apcnn_lateral_fwd: 16-byte alignment");
  ap_lateral_fwd_kernel<<<grid_1d((size_t)N * 4 * h * w * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(top, lat, out, N, h, w,
                                                                                                      C / 4);
  HK_LAUNCH_CHECK("ap_lateral_fwd_kernel");
  return 0;
}

int hk_apcnn_lateral_bwd(const float* dout, float* dtop, int N, int h, int w, int C, void* stream) {
  HK_REQUIRE(dout && dtop, HK_ERR_ARG, "hk_apcnn_lateral_bwd: null pointer");
  HK_REQUIRE(N > 0 && h > 0 && w > 0 && C > 0 && C % 4 == 0, HK_ERR_ARG, "hk_apcnn_lateral_bwd: N=%d h=%d w=%d C=%d (C %% 4)", N,
             h, w, C);
  HK_REQUIRE(aligned16(dout) && aligned16(dtop), HK_ERR_ALIGN, "hk_apcnn_lateral_bwd: 16-byte alignment");
  ap_lateral_bwd_kernel<<<grid_1d((size_t)N * h * w * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(dout, dtop, N, h, w, C / 4);
  HK_LAUNCH_CHECK("ap_lateral_bwd_kernel");
  return 0;
}

int hk_apcnn_bcast(const float* a, const float* b, float* y, int N, int HW, int C, float scale, void* stream) {
  HK_REQUIRE(b && y, HK_ERR_ARG, "hk_apcnn_bcast: null pointer");
  HK_REQUIRE(N > 0 && HW > 0 && C > 0 && C % 4 == 0, HK_ERR_ARG, "hk_apcnn_bcast: N=%d HW=%d C=%d (C %% 4)", N, HW, C);
  HK_REQUIRE((!a || aligned16(a)) && aligned16(b) && aligned16(y), HK_ERR_ALIGN, "hk_apcnn_bcast: 16-byte alignment");
  ap_bcast_kernel<<<grid_1d((size_t)N * HW * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(a, b, y, N, HW, C / 4, scale);
  HK_LAUNCH_CHECK("ap_bcast_kernel");
  return 0;
}

size_t hk_apcnn_pool_workspace_bytes(int N, int HW, int C) {
  if (N <= 0 || HW <= 0 || C <= 0) return 0;
  const int chunk = pool_chunk(HW);
  return (size_t)N * ((HW + chunk - 1) / chunk) * C * sizeof(float);
}

int hk_apcnn_pool(const float* x, float* y, int N, int HW, int C, float scale, void* workspace, size_t workspace_bytes,
                  void* stream) {
  HK_REQUIRE(x && y, HK_ERR_ARG, "hk_apcnn_pool: null pointer");
  HK_REQUIRE(N > 0 && N <= 65535 && HW > 0 && C > 0 && C % 256 == 0, HK_ERR_ARG, "hk_apcnn_pool: N=%d HW=%d C=%d (C %% 256)", N,
             HW, C);
  HK_REQUIRE(workspace && workspace_bytes >= hk_apcnn_pool_workspace_bytes(N, HW, C), HK_ERR_WORKSPACE,
             "hk_apcnn_pool: workspace too small");
  HK_REQUIRE(aligned16(x) && aligned16(workspace), HK_ERR_ALIGN, "hk_apcnn_pool: 16-byte alignment");
  const int chunk = pool_chunk(HW), chunks = (HW + chunk - 1) / chunk;
  float* part = static_cast<float*>(workspace);
  ap_pool_partial_kernel<false><<<dim3(chunks, N, C / 256), 256, 0, (cudaStream_t)stream>>>(x, nullptr, part, HW, C, chunk, chunks);
  HK_LAUNCH_CHECK("ap_pool_partial_kernel");
  ap_pool_final_kernel<<<grid_1d((size_t)N * C, 256), 256, 0, (cudaStream_t)stream>>>(part, y, nullptr, N, C, chunks, 1, scale);
  HK_LAUNCH_CHECK("ap_pool_final_kernel");
  return 0;
}

size_t hk_apcnn_att_workspace_bytes(int N, int H, int W) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  return ((size_t)N * H * W * 12 + (size_t)N * att_chunks(H, W) * AP_ROW) * sizeof(float);
}

static int att_check(const char* op, int N, int H, int W, int C, const void* ws, size_t ws_bytes) {
  HK_REQUIRE(N > 0 && N <= 65535 && H > 0 && W > 0, HK_ERR_ARG, "%s: N=%d H=%d W=%d", op, N, H, W);
  HK_REQUIRE(C == AP_C, HK_ERR_UNSUPPORTED, "%s: C=%d, the pyramid maps have %d channels", op, C, AP_C);
  HK_REQUIRE(ws && ws_bytes >= hk_apcnn_att_workspace_bytes(N, H, W), HK_ERR_WORKSPACE, "%s: workspace too small", op);
  HK_REQUIRE(aligned16(ws), HK_ERR_ALIGN, "%s: workspace must be 16-byte aligned", op);
  return 0;
}

int hk_apcnn_att_fwd(const float* F, const float* w, const float* bias, float* gate, float* pool_f, float* pool_sf, int N,
                     int H, int W, int C, void* workspace, size_t workspace_bytes, void* stream) {
  HK_REQUIRE(F && w && bias && gate && pool_f && pool_sf, HK_ERR_ARG, "hk_apcnn_att_fwd: null pointer");
  if (int r = att_check("hk_apcnn_att_fwd", N, H, W, C, workspace, workspace_bytes)) return r;
  HK_REQUIRE(aligned16(F), HK_ERR_ALIGN, "hk_apcnn_att_fwd: F must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t P = (size_t)N * H * W;
  const int chunks = (int)att_chunks(H, W);
  float* T = static_cast<float*>(workspace);
  float* part = T + P * 12;
  ap_att_taps_kernel<<<grid_1d((P + 15) / 16 * 32, 256), 256, 0, s>>>(F, w, T, P);
  HK_LAUNCH_CHECK("ap_att_taps_kernel");
  ap_att_pool_kernel<<<dim3(chunks, N), 256, 0, s>>>(F, T, bias, gate, part, H, W, chunks);
  HK_LAUNCH_CHECK("ap_att_pool_kernel");
  ap_pool_final_kernel<<<grid_1d((size_t)N * 2 * AP_C, 256), 256, 0, s>>>(part, pool_f, pool_sf, N, AP_C, chunks, 2,
                                                                         1.f / (float)(H * W));
  HK_LAUNCH_CHECK("ap_pool_final_kernel");
  return 0;
}

int hk_apcnn_att_bwd(const float* F, const float* w, const float* gate, const float* dpool_f, const float* dpool_sf, float* dF,
                     float* dw, float* db, int N, int H, int W, int C, void* workspace, size_t workspace_bytes, void* stream) {
  HK_REQUIRE(F && w && gate && dpool_sf && dF && dw && db, HK_ERR_ARG, "hk_apcnn_att_bwd: null pointer");
  if (int r = att_check("hk_apcnn_att_bwd", N, H, W, C, workspace, workspace_bytes)) return r;
  HK_REQUIRE(aligned16(F) && aligned16(dF) && aligned16(dpool_sf) && (!dpool_f || aligned16(dpool_f)), HK_ERR_ALIGN,
             "hk_apcnn_att_bwd: 16-byte alignment");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t P = (size_t)N * H * W;
  const int chunks = (int)att_chunks(H, W);
  float* dz = static_cast<float*>(workspace);
  float* part = dz + P * 12;
  ap_att_dz_kernel<<<grid_1d((P + 3) / 4 * 32, 256), 256, 0, s>>>(F, gate, dpool_sf, dz, P, H * W);
  HK_LAUNCH_CHECK("ap_att_dz_kernel");
  ap_att_bwd_kernel<<<dim3(chunks, N), 256, 0, s>>>(F, w, gate, dz, dpool_f, dpool_sf, dF, part, H, W, chunks);
  HK_LAUNCH_CHECK("ap_att_bwd_kernel");
  ap_att_bwd_final_kernel<<<(AP_DW + 1 + 127) / 128, 128, 0, s>>>(part, dw, db, N * chunks);
  HK_LAUNCH_CHECK("ap_att_bwd_final_kernel");
  return 0;
}

int hk_apcnn_roi(const float* g3, const float* g4, const float* g5, const int* windows, const unsigned char* keep, float* boxes,
                 int* counts, int N, int H3, int W3, int img_h, int img_w, void* stream) {
  HK_REQUIRE(g3 && g4 && g5 && windows && keep && boxes && counts, HK_ERR_ARG, "hk_apcnn_roi: null pointer");
  HK_REQUIRE(N > 0 && N <= 65535 && H3 > 0 && W3 > 0 && H3 % 4 == 0 && W3 % 4 == 0 && img_h > 0 && img_w > 0, HK_ERR_ARG,
             "hk_apcnn_roi: N=%d H3=%d W3=%d (multiples of 4) image %dx%d", N, H3, W3, img_h, img_w);
  const size_t smem = (size_t)H3 * W3 * (sizeof(float) + 1);
  HK_REQUIRE(smem <= 48 * 1024, HK_ERR_UNSUPPORTED, "hk_apcnn_roi: a %dx%d level-3 map does not fit in shared memory", H3, W3);
  RoiArgs a;
  a.g[0] = g3; a.g[1] = g4; a.g[2] = g5;
  for (int l = 0; l < 3; ++l) {
    const int h = H3 >> l, w = W3 >> l;
    for (int k = 0; k < 4; ++k) a.win[l][k] = windows[l * 4 + k];
    HK_REQUIRE(0 <= a.win[l][0] && a.win[l][0] < a.win[l][1] && a.win[l][1] <= h && 0 <= a.win[l][2] && a.win[l][2] < a.win[l][3] &&
                   a.win[l][3] <= w,
               HK_ERR_ARG, "hk_apcnn_roi: the central window of level %d is empty or outside its %dx%d map", l + 3, h, w);
  }
  ap_roi_kernel<<<dim3(N, 3), 256, smem, (cudaStream_t)stream>>>(a, keep, boxes, counts, H3, W3, img_h, img_w);
  HK_LAUNCH_CHECK("ap_roi_kernel");
  return 0;
}

int hk_apcnn_refine_fwd(const float* x, const float* boxes, const int* counts, const float* draws, float* y, int* meta, int N,
                        int H, int W, int C, void* stream) {
  HK_REQUIRE(x && boxes && counts && y && meta, HK_ERR_ARG, "hk_apcnn_refine_fwd: null pointer");
  HK_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, HK_ERR_ARG, "hk_apcnn_refine_fwd: N=%d H=%d W=%d C=%d (C %% 4)", N,
             H, W, C);
  HK_REQUIRE(aligned16(x) && aligned16(y), HK_ERR_ALIGN, "hk_apcnn_refine_fwd: 16-byte alignment");
  ap_refine_meta_kernel<<<(N + 63) / 64, 64, 0, (cudaStream_t)stream>>>(boxes, counts, draws, meta, N, H, W);
  HK_LAUNCH_CHECK("ap_refine_meta_kernel");
  ap_refine_fwd_kernel<<<grid_1d((size_t)N * H * W * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(x, meta, y, N, H, W, C / 4);
  HK_LAUNCH_CHECK("ap_refine_fwd_kernel");
  return 0;
}

int hk_apcnn_refine_bwd(const float* dy, const int* meta, float* dx, int N, int H, int W, int C, void* stream) {
  HK_REQUIRE(dy && meta && dx, HK_ERR_ARG, "hk_apcnn_refine_bwd: null pointer");
  HK_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, HK_ERR_ARG, "hk_apcnn_refine_bwd: N=%d H=%d W=%d C=%d (C %% 4)", N,
             H, W, C);
  HK_REQUIRE(aligned16(dy) && aligned16(dx), HK_ERR_ALIGN, "hk_apcnn_refine_bwd: 16-byte alignment");
  ap_refine_bwd_kernel<<<grid_1d((size_t)N * H * W * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(dy, meta, dx, N, H, W, C / 4);
  HK_LAUNCH_CHECK("ap_refine_bwd_kernel");
  return 0;
}

int hk_apcnn_mix_fwd(const float* z, const float* pm, const float* psf, float* v, float* ch, int N, int C, void* stream) {
  HK_REQUIRE(z && pm && psf && v && ch, HK_ERR_ARG, "hk_apcnn_mix_fwd: null pointer");
  HK_REQUIRE(N > 0 && C > 0, HK_ERR_ARG, "hk_apcnn_mix_fwd: N=%d C=%d", N, C);
  ap_mix_fwd_kernel<<<grid_1d((size_t)N * C, 256), 256, 0, (cudaStream_t)stream>>>(z, pm, psf, v, ch, N * C);
  HK_LAUNCH_CHECK("ap_mix_fwd_kernel");
  return 0;
}

int hk_apcnn_mix_bwd(const float* z, const float* pm, const float* ch, const float* dv, float* dz, float* dpm, int N, int C,
                     void* stream) {
  HK_REQUIRE(z && pm && ch && dv && dz && dpm, HK_ERR_ARG, "hk_apcnn_mix_bwd: null pointer");
  HK_REQUIRE(N > 0 && C > 0, HK_ERR_ARG, "hk_apcnn_mix_bwd: N=%d C=%d", N, C);
  ap_mix_bwd_kernel<<<grid_1d((size_t)N * C, 256), 256, 0, (cudaStream_t)stream>>>(z, pm, ch, dv, dz, dpm, N * C);
  HK_LAUNCH_CHECK("ap_mix_bwd_kernel");
  return 0;
}

int hk_apcnn_mask_cat(const float* g3, const float* g4, const float* g5, float* out, int N, int H3, int W3, void* stream) {
  HK_REQUIRE(g3 && g4 && g5 && out, HK_ERR_ARG, "hk_apcnn_mask_cat: null pointer");
  HK_REQUIRE(N > 0 && H3 > 0 && W3 > 0 && H3 % 4 == 0 && W3 % 4 == 0, HK_ERR_ARG, "hk_apcnn_mask_cat: N=%d H3=%d W3=%d", N, H3,
             W3);
  ap_mask_cat_kernel<<<grid_1d((size_t)N * 3 * H3 * W3, 256), 256, 0, (cudaStream_t)stream>>>(g3, g4, g5, out, N, H3, W3);
  HK_LAUNCH_CHECK("ap_mask_cat_kernel");
  return 0;
}

}  // extern "C"
