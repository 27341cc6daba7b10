// Support kernels of the ResNet-50 v1.5 trunk (reference model/backbone/resnet.py:89-252) around the tensor-core
// convolutions: 7x7/s2 stem patch extraction, train-mode BatchNorm2d (batch statistics, running-stat update,
// fused residual add + ReLU) forward/backward, MaxPool2d(3,2,1), stride-2 sub/up-sampling, 1x1-conv weight
// gradient (split-K GEMM), and the elementwise layers the methods share (in-place add, ReLU / ELU, NCHW <-> NHWC).
// All activations NHWC fp32; every kernel here is HBM-bound.
#include "common.cuh"
#include "host.h"
#include "gemm.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

// ------------------------------------------------------------------------------------------------ stem (resnet.py:176)
// X147[pix][ci*49 + kh*7 + kw] = x[n][ci][2*ho+kh-3][2*wo+kw-3] (0 outside), columns 147..159 = 0; tf32-rounded
__global__ void stem_im2col_kernel(const float* __restrict__ x, float* __restrict__ o, int N, int H, int W, int Ho,
                                   int Wo, int round) {
  const long long total = (long long)N * Ho * Wo * 40;   // 40 float4 per pixel
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % 40);
    const long long pix = i / 40;
    const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho), n = (int)(pix / ((long long)Wo * Ho));
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int col = q * 4 + e;
      float t = 0.f;
      if (col < 147) {
        const int ci = col / 49, r = col % 49, kh = r / 7, kw = r % 7;
        const int hh = 2 * ho + kh - 3, ww = 2 * wo + kw - 3;
        if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
          t = __ldg(x + (((size_t)n * 3 + ci) * H + hh) * W + ww);
          if (round) t = tf32_round(t);
        }
      }
      v[e] = t;
    }
    reinterpret_cast<float4*>(o)[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}
__global__ void pack_stem_weights_kernel(const float* __restrict__ w, float* __restrict__ o, int Cout, int round) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Cout * 160) return;
  const int co = i / 160, c = i % 160;
  o[i] = c < 147 ? (round ? tf32_round(w[co * 147 + c]) : w[co * 147 + c]) : 0.f;
}

// ------------------------------------------------------------------------------------------------ BatchNorm2d (train)
// per-block partial column sums of d = x - x[0] and d^2 over a slab of pixels:  part[blk][0][c], part[blk][1][c].
// Summing x and x^2 directly would lose the variance to cancellation in E[x^2] - mean^2 when a channel's mean is large
// against its spread (at mean = 100 sigma, up to 2e-3 of invstd); the shift by the channel's first value keeps d at the
// spread's scale, and x - x[0] is exact for values within a factor 2 of each other.
__global__ void bn_stats_partial_kernel(const float* __restrict__ x, float* __restrict__ part, long long P, int C) {
  extern __shared__ float sm[];   // [2][plan][C4*4]
  const int C4 = C / 4;
  const int clanes = C4 < (int)blockDim.x ? C4 : (int)blockDim.x;
  const int plan = (int)blockDim.x / clanes;
  const int cl = threadIdx.x % clanes, pl = threadIdx.x / clanes;
  const long long per = (P + gridDim.x - 1) / gridDim.x;
  const long long p0 = blockIdx.x * per, p1 = (p0 + per < P) ? p0 + per : P;
  for (int c4 = cl; c4 < C4; c4 += clanes) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
    if (pl < plan) {
      const float4 k = __ldg(reinterpret_cast<const float4*>(x) + c4);
#pragma unroll 8
      for (long long p = p0 + pl; p < p1; p += plan) {
        float4 v = __ldg(reinterpret_cast<const float4*>(x + p * C) + c4);
        v.x -= k.x; v.y -= k.y; v.z -= k.z; v.w -= k.w;
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        q.x = fmaf(v.x, v.x, q.x); q.y = fmaf(v.y, v.y, q.y); q.z = fmaf(v.z, v.z, q.z); q.w = fmaf(v.w, v.w, q.w);
      }
      reinterpret_cast<float4*>(sm + (size_t)pl * C)[c4] = s;
      reinterpret_cast<float4*>(sm + (size_t)(plan + pl) * C)[c4] = q;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f, q = 0.f;
    for (int k = 0; k < plan; ++k) { s += sm[(size_t)k * C + c]; q += sm[(size_t)(plan + k) * C + c]; }
    part[((size_t)blockIdx.x * 2) * C + c] = s;
    part[((size_t)blockIdx.x * 2 + 1) * C + c] = q;
  }
}
// mean / invstd (biased variance) + running-stat update with the unbiased variance (nn.BatchNorm2d, momentum 0.1), from
// the shifted sums of bn_stats_partial_kernel: mean = x[0] + E[d], var = E[d^2] - E[d]^2
__global__ void bn_stats_finalize_kernel(const float* __restrict__ x, const float* __restrict__ part, int nblk, long long P,
                                         int C, float eps, float momentum, float* __restrict__ mean,
                                         float* __restrict__ invstd, float* __restrict__ rmean, float* __restrict__ rvar) {
  // block = 32 channels x 32 partial-row lanes: lanes run along channels (coalesced 128 B reads of the partial rows)
  __shared__ float red[2][32][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  float s = 0.f, q = 0.f;
  if (c < C) {
#pragma unroll 4
    for (int b = w; b < nblk; b += 32) { s += part[((size_t)b * 2) * C + c]; q += part[((size_t)b * 2 + 1) * C + c]; }
  }
  red[0][w][lane] = s; red[1][w][lane] = q;
  __syncthreads();
  if (w != 0 || c >= C) return;
  double sd = 0.0, qd = 0.0;
  for (int k = 0; k < 32; ++k) { sd += (double)red[0][k][lane]; qd += (double)red[1][k][lane]; }
  const double md = sd / (double)P;
  double var = qd / (double)P - md * md;
  if (var < 0.0) var = 0.0;
  const double m = (double)x[c] + md;
  mean[c] = (float)m;
  invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
  if (rmean) {
    const double unb = P > 1 ? var * (double)P / (double)(P - 1) : var;
    rmean[c] = (1.f - momentum) * rmean[c] + momentum * (float)m;
    rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)unb;
  }
}
// y = [relu]( (x-mean)*invstd*gamma + beta [+ residual] ), tf32-rounded (it feeds the next MMA)
__global__ void bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                const float* __restrict__ invstd, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const float* __restrict__ res, float* __restrict__ y,
                                size_t total4, int C4, int relu, int round) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    const float4 m = reinterpret_cast<const float4*>(mean)[c4], is = reinterpret_cast<const float4*>(invstd)[c4];
    const float4 g = reinterpret_cast<const float4*>(gamma)[c4], b = reinterpret_cast<const float4*>(beta)[c4];
    float4 o;
    o.x = fmaf((v.x - m.x) * is.x, g.x, b.x); o.y = fmaf((v.y - m.y) * is.y, g.y, b.y);
    o.z = fmaf((v.z - m.z) * is.z, g.z, b.z); o.w = fmaf((v.w - m.w) * is.w, g.w, b.w);
    if (res) {
      const float4 r = reinterpret_cast<const float4*>(res)[i];
      o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
    }
    if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
    if (round) o = make_float4(tf32_round(o.x), tf32_round(o.y), tf32_round(o.z), tf32_round(o.w));
    reinterpret_cast<float4*>(y)[i] = o;
  }
}
// backward reductions: part[blk][0][c] = sum dy', part[blk][1][c] = sum dy' * xhat,  dy' = dy * (y > 0 if relu)
// relu with gamma/beta given (and no residual in the forward): the ReLU mask is recomputed from x with the forward's own
// expression, so y (a third of the bytes) is not read at all
__global__ void bn_bwd_partial_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                      const float* __restrict__ dy, const float* __restrict__ mean,
                                      const float* __restrict__ invstd, const float* __restrict__ gamma,
                                      const float* __restrict__ beta, float* __restrict__ part, long long P, int C,
                                      int relu) {
  extern __shared__ float sm[];
  const int C4 = C / 4;
  const int clanes = C4 < (int)blockDim.x ? C4 : (int)blockDim.x;
  const int plan = (int)blockDim.x / clanes;
  const int cl = threadIdx.x % clanes, pl = threadIdx.x / clanes;
  const long long per = (P + gridDim.x - 1) / gridDim.x;
  const long long p0 = blockIdx.x * per, p1 = (p0 + per < P) ? p0 + per : P;
  for (int c4 = cl; c4 < C4; c4 += clanes) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
    if (pl < plan) {
      const float4 m = reinterpret_cast<const float4*>(mean)[c4], is = reinterpret_cast<const float4*>(invstd)[c4];
      float4 ga = make_float4(0.f, 0.f, 0.f, 0.f), be = ga;
      if (relu && beta) { ga = reinterpret_cast<const float4*>(gamma)[c4]; be = reinterpret_cast<const float4*>(beta)[c4]; }
#pragma unroll 4
      for (long long p = p0 + pl; p < p1; p += plan) {
        float4 g = __ldg(reinterpret_cast<const float4*>(dy + p * C) + c4);
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + p * C) + c4);
        if (relu && beta) {
          g.x = fmaf((v.x - m.x) * is.x, ga.x, be.x) > 0.f ? g.x : 0.f; g.y = fmaf((v.y - m.y) * is.y, ga.y, be.y) > 0.f ? g.y : 0.f;
          g.z = fmaf((v.z - m.z) * is.z, ga.z, be.z) > 0.f ? g.z : 0.f; g.w = fmaf((v.w - m.w) * is.w, ga.w, be.w) > 0.f ? g.w : 0.f;
        } else if (relu) {
          const float4 o = __ldg(reinterpret_cast<const float4*>(y + p * C) + c4);
          g.x = o.x > 0.f ? g.x : 0.f; g.y = o.y > 0.f ? g.y : 0.f; g.z = o.z > 0.f ? g.z : 0.f; g.w = o.w > 0.f ? g.w : 0.f;
        }
        s.x += g.x; s.y += g.y; s.z += g.z; s.w += g.w;
        q.x = fmaf(g.x, (v.x - m.x) * is.x, q.x); q.y = fmaf(g.y, (v.y - m.y) * is.y, q.y);
        q.z = fmaf(g.z, (v.z - m.z) * is.z, q.z); q.w = fmaf(g.w, (v.w - m.w) * is.w, q.w);
      }
      reinterpret_cast<float4*>(sm + (size_t)pl * C)[c4] = s;
      reinterpret_cast<float4*>(sm + (size_t)(plan + pl) * C)[c4] = q;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f, q = 0.f;
    for (int k = 0; k < plan; ++k) { s += sm[(size_t)k * C + c]; q += sm[(size_t)(plan + k) * C + c]; }
    part[((size_t)blockIdx.x * 2) * C + c] = s;
    part[((size_t)blockIdx.x * 2 + 1) * C + c] = q;
  }
}
__global__ void bn_bwd_finalize_kernel(const float* __restrict__ part, int nblk, int C, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta) {
  // block = 32 channels x 32 partial-row lanes: lanes run along channels (coalesced 128 B reads of the partial rows)
  __shared__ float red[2][32][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  float s = 0.f, q = 0.f;
  if (c < C) {
#pragma unroll 4
    for (int b = w; b < nblk; b += 32) { s += part[((size_t)b * 2) * C + c]; q += part[((size_t)b * 2 + 1) * C + c]; }
  }
  red[0][w][lane] = s; red[1][w][lane] = q;
  __syncthreads();
  if (w != 0 || c >= C) return;
  double sd = 0.0, qd = 0.0;
  for (int k = 0; k < 32; ++k) { sd += (double)red[0][k][lane]; qd += (double)red[1][k][lane]; }
  dbeta[c] = (float)sd;
  dgamma[c] = (float)qd;
}
// dx = gamma*invstd*(dy' - dbeta/P - xhat*dgamma/P)  (tf32-rounded: operand of dgrad/wgrad);  dres = dy' (optional)
__global__ void bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                    const float* __restrict__ dy, const float* __restrict__ mean,
                                    const float* __restrict__ invstd, const float* __restrict__ gamma,
                                    const float* __restrict__ dgamma, const float* __restrict__ dbeta,
                                    const float* __restrict__ beta, float* __restrict__ dx, float* __restrict__ dres,
                                    size_t total4, int C4, float invP, int relu, int round) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    float4 g = reinterpret_cast<const float4*>(dy)[i];
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    const float4 m = reinterpret_cast<const float4*>(mean)[c4], is = reinterpret_cast<const float4*>(invstd)[c4];
    const float4 ga = reinterpret_cast<const float4*>(gamma)[c4];
    if (relu && beta) {
      const float4 be = reinterpret_cast<const float4*>(beta)[c4];
      g.x = fmaf((v.x - m.x) * is.x, ga.x, be.x) > 0.f ? g.x : 0.f; g.y = fmaf((v.y - m.y) * is.y, ga.y, be.y) > 0.f ? g.y : 0.f;
      g.z = fmaf((v.z - m.z) * is.z, ga.z, be.z) > 0.f ? g.z : 0.f; g.w = fmaf((v.w - m.w) * is.w, ga.w, be.w) > 0.f ? g.w : 0.f;
    } else if (relu) {
      const float4 o = reinterpret_cast<const float4*>(y)[i];
      g.x = o.x > 0.f ? g.x : 0.f; g.y = o.y > 0.f ? g.y : 0.f; g.z = o.z > 0.f ? g.z : 0.f; g.w = o.w > 0.f ? g.w : 0.f;
    }
    if (dres) reinterpret_cast<float4*>(dres)[i] = g;
    const float4 dg = reinterpret_cast<const float4*>(dgamma)[c4], db = reinterpret_cast<const float4*>(dbeta)[c4];
    float4 o;
    o.x = ga.x * is.x * (g.x - db.x * invP - (v.x - m.x) * is.x * dg.x * invP);
    o.y = ga.y * is.y * (g.y - db.y * invP - (v.y - m.y) * is.y * dg.y * invP);
    o.z = ga.z * is.z * (g.z - db.z * invP - (v.z - m.z) * is.z * dg.z * invP);
    o.w = ga.w * is.w * (g.w - db.w * invP - (v.w - m.w) * is.w * dg.w * invP);
    if (round) o = make_float4(tf32_round(o.x), tf32_round(o.y), tf32_round(o.z), tf32_round(o.w));
    reinterpret_cast<float4*>(dx)[i] = o;
  }
}

// ------------------------------------------------------------------------------------------------ MaxPool2d(3, 2, 1)
// forward also records, per output element, which of the 9 window positions held the first maximum (PyTorch routing)
__global__ void maxpool3x3s2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y,
                                        unsigned char* __restrict__ arg, int N, int H, int W, int C, int Ho, int Wo) {
  const int C4 = C / 4;
  const size_t total = (size_t)N * Ho * Wo * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    size_t p = i / C4;
    const int wo = p % Wo; p /= Wo;
    const int ho = p % Ho;
    const int n = p / Ho;
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    uchar4 am = make_uchar4(0, 0, 0, 0);
    for (int kh = 0; kh < 3; ++kh) {
      const int hh = 2 * ho + kh - 1;
      if (hh < 0 || hh >= H) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int ww = 2 * wo + kw - 1;
        if (ww < 0 || ww >= W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + (((size_t)n * H + hh) * W + ww) * C) + c4);
        const unsigned char k = (unsigned char)(kh * 3 + kw);
        if (v.x > m.x) { m.x = v.x; am.x = k; }
        if (v.y > m.y) { m.y = v.y; am.y = k; }
        if (v.z > m.z) { m.z = v.z; am.z = k; }
        if (v.w > m.w) { m.w = v.w; am.w = k; }
      }
    }
    reinterpret_cast<float4*>(y)[i] = m;
    if (arg) reinterpret_cast<uchar4*>(arg)[i] = am;
  }
}
// gather form (no atomics): an input pixel belongs to <= 2x2 windows; it receives dy of those whose recorded arg-max is it
__global__ void maxpool3x3s2_bwd_kernel(const unsigned char* __restrict__ arg, const float* __restrict__ dy,
                                        float* __restrict__ dx, int N, int H, int W, int C, int Ho, int Wo) {
  const int C4 = C / 4;
  const size_t total = (size_t)N * H * W * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    size_t p = i / C4;
    const int w = p % W; p /= W;
    const int h = p % H;
    const int n = p / H;
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    const int ho0 = h >> 1, wo0 = w >> 1;   // windows ho with 2ho-1 <= h <= 2ho+1: ho0 (+1 if h odd)
    for (int dh = 0; dh <= (h & 1); ++dh) {
      const int ho = ho0 + dh;
      if (ho >= Ho) continue;
      const int kh = h - 2 * ho + 1;
      for (int dw = 0; dw <= (w & 1); ++dw) {
        const int wo = wo0 + dw;
        if (wo >= Wo) continue;
        const unsigned char k = (unsigned char)(kh * 3 + (w - 2 * wo + 1));
        const size_t oi = (((size_t)n * Ho + ho) * Wo + wo) * C4 + c4;
        const uchar4 am = __ldg(reinterpret_cast<const uchar4*>(arg) + oi);
        const float4 d = __ldg(reinterpret_cast<const float4*>(dy) + oi);
        if (am.x == k) g.x += d.x;
        if (am.y == k) g.y += d.y;
        if (am.z == k) g.z += d.z;
        if (am.w == k) g.w += d.w;
      }
    }
    reinterpret_cast<float4*>(dx)[i] = g;
  }
}

// ------------------------------------------------------------------------------------------------ stride-2 helpers
__global__ void subsample2_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int H, int W, int C4) {
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const size_t total = (size_t)N * Ho * Wo * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    size_t p = i / C4;
    const int wo = p % Wo; p /= Wo;
    const int ho = p % Ho;
    const int n = p / Ho;
    reinterpret_cast<float4*>(y)[i] = reinterpret_cast<const float4*>(x)[(((size_t)n * H + 2 * ho) * W + 2 * wo) * C4 + c4];
  }
}
// x[n][h][w] = (h,w even) ? y[n][h/2][w/2] : 0
__global__ void upsample2_zero_kernel(const float* __restrict__ y, float* __restrict__ x, int N, int H, int W, int C4) {
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const size_t total = (size_t)N * H * W * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    size_t p = i / C4;
    const int w = p % W; p /= W;
    const int h = p % H;
    const int n = p / H;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (((h | w) & 1) == 0) v = reinterpret_cast<const float4*>(y)[(((size_t)n * Ho + h / 2) * Wo + w / 2) * C4 + c4];
    reinterpret_cast<float4*>(x)[i] = v;
  }
}
__global__ void add_inplace_kernel(float* __restrict__ a, const float* __restrict__ b, size_t n4) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 u = reinterpret_cast<float4*>(a)[i];
    const float4 v = reinterpret_cast<const float4*>(b)[i];
    u.x += v.x; u.y += v.y; u.z += v.z; u.w += v.w;
    reinterpret_cast<float4*>(a)[i] = u;
  }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int HW, int C) {
  const size_t total = (size_t)N * HW * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int p = i % HW;
    const int c = (i / HW) % C;
    const int n = i / ((size_t)HW * C);
    y[i] = x[((size_t)n * HW + p) * C + c];
  }
}
// ReLU (elu = 0) or ELU with alpha 1 (elu = 1)
__global__ void act_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n, int elu) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    y[i] = v > 0.f ? v : (elu ? expm1f(v) : 0.f);
  }
}

// from the output: ReLU passes where y > 0; ELU (alpha 1) has slope y + 1 where y <= 0
__global__ void act_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, float* __restrict__ dx, size_t n,
                               int elu) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = y[i];
    dx[i] = v > 0.f ? dy[i] : (elu ? dy[i] * (v + 1.f) : 0.f);
  }
}
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int HW, int C) {
  const size_t total = (size_t)N * HW * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = i % C;
    const int p = (i / C) % HW;
    const int n = i / ((size_t)HW * C);
    y[i] = x[((size_t)n * C + c) * HW + p];
  }
}

static int bn_blocks(long long P) {
  long long b = (P + 255) / 256;
  if (b > 592) b = 592;      // 4 blocks per SM: the partial-sum kernels need ~8 MB of loads in flight to reach HBM bandwidth
  if (b < 1) b = 1;
  return (int)b;
}
// split-K factor of the 1x1-conv weight gradient dW[Cout][K] = dY^T . X over P pixels: just enough splits to fill the SMs about
// twice with 128 x BN output tiles (the partial sums cost S x Cout x K floats of write + read: with the former "as many as divide
// P" rule a 2048x512 layer moved 0.4 GB per call through the reduction), each split at least 64 pixels long; S divides P.
static int kc_splits(long long P, int Cout, int K) {
  const int BN = K <= 64 ? 64 : (K <= 128 ? 128 : 256);
  const long long tiles = (long long)((Cout + 127) / 128) * ((K + BN - 1) / BN);
  long long target = (296 + tiles - 1) / tiles;
  if (target > 296) target = 296;
  for (long long S = target; S > 1; --S)
    if (P % S == 0 && P / S >= 64) return (int)S;
  return 1;
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_stem_im2col(const float* x_nchw, float* x147, int N, int H, int W, void* stream) {
  HK_REQUIRE(x_nchw && x147, HK_ERR_ARG, "hk_stem_im2col: null pointer");
  const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
  stem_im2col_kernel<<<grid_1d((size_t)N * Ho * Wo * 40, 256), 256, 0, (cudaStream_t)stream>>>(x_nchw, x147, N, H, W, Ho, Wo, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("stem_im2col_kernel");
  return 0;
}
int hk_pack_stem_weights(const float* w, float* w147, int Cout, void* stream) {
  HK_REQUIRE(w && w147, HK_ERR_ARG, "hk_pack_stem_weights: null pointer");
  pack_stem_weights_kernel<<<(Cout * 160 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w, w147, Cout, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("pack_stem_weights_kernel");
  return 0;
}

size_t hk_bn_workspace_bytes(long long P, int C) { return (size_t)bn_blocks(P) * 2 * C * sizeof(float); }

int hk_bn_fwd(const float* x, const float* gamma, const float* beta, const float* residual, float* y, float* save_mean,
              float* save_invstd, float* running_mean, float* running_var, float momentum, float eps, long long P, int C,
              int relu, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  HK_REQUIRE(x && gamma && beta && y && save_mean && save_invstd, HK_ERR_ARG, "hk_bn_fwd: null pointer");
  HK_REQUIRE(C % 4 == 0 && P > 0, HK_ERR_UNSUPPORTED, "hk_bn_fwd: C=%d must be a multiple of 4", C);
  HK_REQUIRE(workspace && workspace_bytes >= hk_bn_workspace_bytes(P, C), HK_ERR_WORKSPACE, "hk_bn_fwd: workspace too small");
  float* part = static_cast<float*>(workspace);
  const int nb = bn_blocks(P);
  const int C4 = C / 4, clanes = C4 < 256 ? C4 : 256, plan = 256 / clanes;
  bn_stats_partial_kernel<<<nb, 256, (size_t)2 * plan * C * sizeof(float), st>>>(x, part, P, C);
  HK_LAUNCH_CHECK("bn_stats_partial_kernel");
  bn_stats_finalize_kernel<<<(C + 31) / 32, 1024, 0, st>>>(x, part, nb, P, C, eps, momentum, save_mean, save_invstd,
                                                         running_mean, running_var);
  HK_LAUNCH_CHECK("bn_stats_finalize_kernel");
  bn_apply_kernel<<<grid_1d((size_t)P * C4, 256), 256, 0, st>>>(x, save_mean, save_invstd, gamma, beta, residual, y,
                                                                (size_t)P * C4, C4, relu, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("bn_apply_kernel");
  return 0;
}

/* eval-mode / given-statistics apply: y = [relu]((x-mean)*invstd*gamma + beta [+ residual]) */
int hk_bn_apply(const float* x, const float* mean, const float* invstd, const float* gamma, const float* beta,
                const float* residual, float* y, long long P, int C, int relu, void* stream_) {
  HK_REQUIRE(x && mean && invstd && gamma && beta && y && C % 4 == 0, HK_ERR_ARG, "hk_bn_apply: bad args");
  bn_apply_kernel<<<grid_1d((size_t)P * (C / 4), 256), 256, 0, (cudaStream_t)stream_>>>(x, mean, invstd, gamma, beta, residual, y,
                                                                                        (size_t)P * (C / 4), C / 4, relu, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("bn_apply_kernel");
  return 0;
}

int hk_bn_bwd_ex(const float* x, const float* y, const float* dy, const float* gamma, const float* beta_for_mask,
                 const float* save_mean, const float* save_invstd, float* dx, float* dres, float* dgamma, float* dbeta,
                 long long P, int C, int relu, void* workspace, size_t workspace_bytes, void* stream_);
int hk_bn_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* save_mean,
              const float* save_invstd, float* dx, float* dres, float* dgamma, float* dbeta, long long P, int C, int relu,
              void* workspace, size_t workspace_bytes, void* stream_) {
  return hk_bn_bwd_ex(x, y, dy, gamma, nullptr, save_mean, save_invstd, dx, dres, dgamma, dbeta, P, C, relu, workspace,
                      workspace_bytes, stream_);
}
}  // extern "C"

// The backward of both BatchNorm modes: the batch-statistics one (frozen = 0) and the one on constant statistics (frozen = 1),
// whose dx lacks the two terms through the batch mean and variance: the apply kernel then runs with invP = 0.
static int bn_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* beta_for_mask,
                  const float* save_mean, const float* save_invstd, float* dx, float* dres, float* dgamma, float* dbeta,
                  long long P, int C, int relu, void* workspace, size_t workspace_bytes, void* stream_, int frozen) {
  cudaStream_t st = (cudaStream_t)stream_;
  const float* beta = relu ? beta_for_mask : nullptr;
  HK_REQUIRE(x && dy && gamma && save_mean && save_invstd && dx && dgamma && dbeta && (!relu || y || beta), HK_ERR_ARG,
             "hk_bn_bwd: null pointer");
  HK_REQUIRE(C % 4 == 0 && P > 0, HK_ERR_UNSUPPORTED, "hk_bn_bwd: C=%d must be a multiple of 4", C);
  HK_REQUIRE(workspace && workspace_bytes >= hk_bn_workspace_bytes(P, C), HK_ERR_WORKSPACE, "hk_bn_bwd: workspace too small");
  float* part = static_cast<float*>(workspace);
  const int nb = bn_blocks(P);
  const int C4 = C / 4, clanes = C4 < 256 ? C4 : 256, plan = 256 / clanes;
  bn_bwd_partial_kernel<<<nb, 256, (size_t)2 * plan * C * sizeof(float), st>>>(x, y, dy, save_mean, save_invstd, gamma, beta, part, P,
                                                                               C, relu);
  HK_LAUNCH_CHECK("bn_bwd_partial_kernel");
  bn_bwd_finalize_kernel<<<(C + 31) / 32, 1024, 0, st>>>(part, nb, C, dgamma, dbeta);
  HK_LAUNCH_CHECK("bn_bwd_finalize_kernel");
  bn_bwd_apply_kernel<<<grid_1d((size_t)P * C4, 256), 256, 0, st>>>(x, y, dy, save_mean, save_invstd, gamma, dgamma, dbeta, beta,
                                                                    dx, dres, (size_t)P * C4, C4, frozen ? 0.f : 1.f / (float)P, relu,
                                                                    precise() ? 0 : 1);
  HK_LAUNCH_CHECK("bn_bwd_apply_kernel");
  return 0;
}

extern "C" {

int hk_bn_bwd_ex(const float* x, const float* y, const float* dy, const float* gamma, const float* beta_for_mask,
                 const float* save_mean, const float* save_invstd, float* dx, float* dres, float* dgamma, float* dbeta,
                 long long P, int C, int relu, void* workspace, size_t workspace_bytes, void* stream_) {
  return bn_bwd(x, y, dy, gamma, beta_for_mask, save_mean, save_invstd, dx, dres, dgamma, dbeta, P, C, relu, workspace,
                workspace_bytes, stream_, 0);
}
int hk_bn_bwd_frozen(const float* x, const float* y, const float* dy, const float* gamma, const float* beta_for_mask,
                     const float* mean, const float* invstd, float* dx, float* dres, float* dgamma, float* dbeta, long long P,
                     int C, int relu, void* workspace, size_t workspace_bytes, void* stream_) {
  return bn_bwd(x, y, dy, gamma, beta_for_mask, mean, invstd, dx, dres, dgamma, dbeta, P, C, relu, workspace, workspace_bytes,
                stream_, 1);
}

int hk_maxpool3x3s2_fwd(const float* x, float* y, unsigned char* argmax, int N, int H, int W, int C, void* stream) {
  HK_REQUIRE(x && y && C % 4 == 0, HK_ERR_ARG, "hk_maxpool3x3s2_fwd: bad args");
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  maxpool3x3s2_fwd_kernel<<<grid_1d((size_t)N * Ho * Wo * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(x, y, argmax, N, H, W, C, Ho, Wo);
  HK_LAUNCH_CHECK("maxpool3x3s2_fwd_kernel");
  return 0;
}
int hk_maxpool3x3s2_bwd(const unsigned char* argmax, const float* dy, float* dx, int N, int H, int W, int C,
                        void* stream) {
  HK_REQUIRE(argmax && dy && dx && C % 4 == 0, HK_ERR_ARG, "hk_maxpool3x3s2_bwd: bad args");
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  maxpool3x3s2_bwd_kernel<<<grid_1d((size_t)N * H * W * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(argmax, dy, dx, N, H, W, C, Ho, Wo);
  HK_LAUNCH_CHECK("maxpool3x3s2_bwd_kernel");
  return 0;
}
int hk_subsample2(const float* x, float* y, int N, int H, int W, int C, void* stream) {
  HK_REQUIRE(x && y && C % 4 == 0, HK_ERR_ARG, "hk_subsample2: bad args");
  subsample2_kernel<<<grid_1d((size_t)N * ((H + 1) / 2) * ((W + 1) / 2) * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(x, y, N, H, W, C / 4);
  HK_LAUNCH_CHECK("subsample2_kernel");
  return 0;
}
int hk_upsample2_zero(const float* y, float* x, int N, int H, int W, int C, void* stream) {
  HK_REQUIRE(x && y && C % 4 == 0, HK_ERR_ARG, "hk_upsample2_zero: bad args");
  upsample2_zero_kernel<<<grid_1d((size_t)N * H * W * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(y, x, N, H, W, C / 4);
  HK_LAUNCH_CHECK("upsample2_zero_kernel");
  return 0;
}
int hk_add_inplace(float* a, const float* b, size_t n, void* stream) {
  HK_REQUIRE(a && b && n % 4 == 0, HK_ERR_ARG, "hk_add_inplace: bad args");
  add_inplace_kernel<<<grid_1d(n / 4, 256), 256, 0, (cudaStream_t)stream>>>(a, b, n / 4);
  HK_LAUNCH_CHECK("add_inplace_kernel");
  return 0;
}
int hk_nhwc_to_nchw(const float* x, float* y, int N, int HW, int C, void* stream) {
  HK_REQUIRE(x && y, HK_ERR_ARG, "hk_nhwc_to_nchw: null pointer");
  nhwc_to_nchw_kernel<<<grid_1d((size_t)N * HW * C, 256), 256, 0, (cudaStream_t)stream>>>(x, y, N, HW, C);
  HK_LAUNCH_CHECK("nhwc_to_nchw_kernel");
  return 0;
}
int hk_nchw_to_nhwc(const float* x, float* y, int N, int HW, int C, void* stream) {
  HK_REQUIRE(x && y, HK_ERR_ARG, "hk_nchw_to_nhwc: null pointer");
  nchw_to_nhwc_kernel<<<grid_1d((size_t)N * HW * C, 256), 256, 0, (cudaStream_t)stream>>>(x, y, N, HW, C);
  HK_LAUNCH_CHECK("nchw_to_nhwc_kernel");
  return 0;
}
int hk_act_fwd(const float* x, float* y, size_t n, int elu, void* stream) {
  HK_REQUIRE(x && y && n > 0, HK_ERR_ARG, "hk_act_fwd: null pointer or n = 0");
  act_fwd_kernel<<<grid_1d(n, 256), 256, 0, (cudaStream_t)stream>>>(x, y, n, elu);
  HK_LAUNCH_CHECK("act_fwd_kernel");
  return 0;
}
int hk_act_bwd(const float* y, const float* dy, float* dx, size_t n, int elu, void* stream) {
  HK_REQUIRE(y && dy && dx && n > 0, HK_ERR_ARG, "hk_act_bwd: null pointer or n = 0");
  act_bwd_kernel<<<grid_1d(n, 256), 256, 0, (cudaStream_t)stream>>>(y, dy, dx, n, elu);
  HK_LAUNCH_CHECK("act_bwd_kernel");
  return 0;
}

/* weight gradient of a matrix-form (1x1 / im2col) convolution: dw [Cout][K] = dY[P][Cout]^T . X[P][K], split-K batched
 * MN-major wgmma GEMM + reduction.  workspace = S * Cout * K floats. */
size_t hk_matconv_wgrad_workspace_bytes(long long P, int K, int Cout) {
  return (size_t)kc_splits(P, Cout, K) * Cout * K * sizeof(float);
}
int hk_matconv_wgrad(const float* x, const float* dy, float* dw, long long P, int K, int Cout, void* workspace,
                     size_t workspace_bytes, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  HK_REQUIRE(x && dy && dw, HK_ERR_ARG, "hk_matconv_wgrad: null pointer");
  HK_REQUIRE(K % 4 == 0 && Cout % 4 == 0, HK_ERR_UNSUPPORTED, "hk_matconv_wgrad: K=%d Cout=%d must be multiples of 4", K, Cout);
  HK_REQUIRE(workspace && workspace_bytes >= hk_matconv_wgrad_workspace_bytes(P, K, Cout), HK_ERR_WORKSPACE,
             "hk_matconv_wgrad: workspace too small");
  return gemm_splitk(dy, 1, Cout, x, 1, K, Cout, K, P, kc_splits(P, Cout, K), static_cast<float*>(workspace), dw, K, K,
                     nullptr, false, st);
}

}  // extern "C"
