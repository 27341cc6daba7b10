// Interp-Parts (reference model/methods/Interp_Parts.py, model/loss/InterpParts_loss.py): the grouping unit
// (Interp_Parts.py:56-122) forward and backward, the part attention head (attconv's 1-channel conv + BatchNorm(1) + ReLU +
// softmax over the parts, :289-291,:349-350) fused with the attention-weighted part sum (:357-361), and the shaping loss
// (InterpParts_loss.py:83-138): the blurred occupancy of each part and the Wasserstein distance of its batch ranking to the
// Beta prior.
//
// Layouts: the trunk map is NHWC x [N, HW, C]; the centres are [K, C]; assign is [N, K, HW] (the reference's [N, K, H, W]);
// the grouped features are [N, K, C], the NHWC input of the 1x1 stacks over P = N*K rows.  Every reduction has one owner and
// a fixed order (partials per pixel tile through a caller-owned workspace, folded in ascending tile / image order), with no
// atomics: the same bits on every run.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

constexpr int IP_MAX_K = 32;             // parts: one register per part in the per-channel loops
constexpr int IP_TP = 32;                // pixels per grouping tile (the tile of the map stays in shared memory)
constexpr int IP_MAX_C = 1536;           // channels: IP_TP x C fp32 of shared memory per tile
constexpr float IP_SUM_EPS = 1e-5f;      // clamp(min=1e-5) of the assignment sum (:108)
constexpr float IP_NORM_EPS = 1e-12f;    // F.normalize's eps (:118)

__device__ __forceinline__ float ip_beta(const float* smooth, int k) { return 1.f / (1.f + expf(-smooth[k])); }

// Loads the tile [IP_TP, C] of image n starting at pixel p0 into xs (zero rows past HW).
__device__ __forceinline__ void ip_load_tile(const float* __restrict__ x, float* xs, int n, int p0, int HW, int C) {
  const int C4 = C >> 2;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  float4* xs4 = reinterpret_cast<float4*>(xs);
  for (int i = threadIdx.x; i < IP_TP * C4; i += blockDim.x) {
    const int p = i / C4, pix = p0 + p;
    xs4[i] = pix < HW ? x4[((size_t)n * HW + pix) * C4 + (i - p * C4)] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// out[k * IP_TP + p] = sum_c xs[p, c] * v[k, c] (dot) or sum_c (xs[p, c] - v[k, c])^2 (!dot) for the pixels of the tile inside
// the map; a warp per (p, k) pair, lanes over float4 channel groups, then the xor tree.
template <bool DOT>
__device__ __forceinline__ void ip_tile_pairs(const float* xs, const float* __restrict__ v, float* out, int valid, int K,
                                              int C) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5, C4 = C >> 2;
  const float4* xs4 = reinterpret_cast<const float4*>(xs);
  const float4* v4 = reinterpret_cast<const float4*>(v);
  for (int j = warp; j < IP_TP * K; j += nw) {
    const int p = j % IP_TP, k = j / IP_TP;
    if (p >= valid) continue;
    float acc = 0.f;
    for (int c4 = lane; c4 < C4; c4 += 32) {
      const float4 a = xs4[p * C4 + c4], b = v4[(size_t)k * C4 + c4];
      if (DOT) {
        acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc); acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
      } else {
        const float t0 = a.x - b.x, t1 = a.y - b.y, t2 = a.z - b.z, t3 = a.w - b.w;
        acc = fmaf(t0, t0, acc); acc = fmaf(t1, t1, acc); acc = fmaf(t2, t2, acc); acc = fmaf(t3, t3, acc);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0) out[k * IP_TP + p] = acc;
  }
}

// Block (tile t, image n).  One read of the tile: D[k, p] = sum_c (x - c_k)^2 directly in fp32, assign = softmax_k(-D / beta)
// (dist and assign stored for the backward and the loss), then the tile's partial qx[k, :] = sum_p assign x[p, :] and
// sum_p assign to the workspace.
__global__ void __launch_bounds__(256) ip_group_fwd_tile_kernel(const float* __restrict__ x, const float* __restrict__ cen,
                                                                const float* __restrict__ smooth, float* __restrict__ assign,
                                                                float* __restrict__ dist, float* __restrict__ pq,
                                                                float* __restrict__ ps, int HW, int K, int C) {
  extern __shared__ float4 ip_smem[];
  float* xs = reinterpret_cast<float*>(ip_smem);
  float* as = xs + (size_t)IP_TP * C;                 // [K][IP_TP]
  const int n = blockIdx.y, t = blockIdx.x, T = gridDim.x, p0 = t * IP_TP;
  const int valid = min(IP_TP, HW - p0);
  ip_load_tile(x, xs, n, p0, HW, C);
  __syncthreads();
  ip_tile_pairs<false>(xs, cen, as, valid, K, C);
  __syncthreads();
  if (threadIdx.x < IP_TP) {
    const int p = threadIdx.x, pix = p0 + p;
    if (p < valid) {
      float m = -INFINITY;
      for (int k = 0; k < K; ++k) m = fmaxf(m, -as[k * IP_TP + p] / ip_beta(smooth, k));
      float s = 0.f;
      for (int k = 0; k < K; ++k) s += expf(-as[k * IP_TP + p] / ip_beta(smooth, k) - m);
      for (int k = 0; k < K; ++k) {
        const float d = as[k * IP_TP + p];
        const float a = expf(-d / ip_beta(smooth, k) - m) / s;
        dist[((size_t)n * K + k) * HW + pix] = d;
        assign[((size_t)n * K + k) * HW + pix] = a;
        as[k * IP_TP + p] = a;
      }
    } else {
      for (int k = 0; k < K; ++k) as[k * IP_TP + p] = 0.f;
    }
  }
  __syncthreads();
  float* pqt = pq + ((size_t)n * T + t) * K * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    for (int k = 0; k < K; ++k) {
      float acc = 0.f;
      for (int p = 0; p < valid; ++p) acc = fmaf(as[k * IP_TP + p], xs[p * C + c], acc);
      pqt[(size_t)k * C + c] = acc;
    }
  if (threadIdx.x < K) {
    float s = 0.f;
    for (int p = 0; p < valid; ++p) s += as[threadIdx.x * IP_TP + p];
    ps[((size_t)n * T + t) * K + threadIdx.x] = s;
  }
}

// Block (k, n): qx = sum over tiles of the partials, s likewise; u = (qx / max(s, 1e-5) - c_k) / sqrt(beta / 2);
// out = u / max(|u|, 1e-12).  qx, s and |u| are saved for the backward.
__global__ void ip_group_fwd_finish_kernel(const float* __restrict__ pq, const float* __restrict__ ps,
                                           const float* __restrict__ cen, const float* __restrict__ smooth,
                                           float* __restrict__ out, float* __restrict__ qx, float* __restrict__ ssum,
                                           float* __restrict__ nrm, int T, int K, int C, int round) {
  __shared__ float red[32];
  const int k = blockIdx.x, n = blockIdx.y;
  float s = 0.f;
  for (int t = 0; t < T; ++t) s += ps[((size_t)n * T + t) * K + k];
  const float S = fmaxf(s, IP_SUM_EPS), sigma = sqrtf(ip_beta(smooth, k) / 2.f);
  float* o = out + ((size_t)n * K + k) * C;
  float* q = qx + ((size_t)n * K + k) * C;
  float ss = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    for (int t = 0; t < T; ++t) acc += pq[(((size_t)n * T + t) * K + k) * C + c];
    q[c] = acc;
    const float u = (acc / S - cen[(size_t)k * C + c]) / sigma;
    o[c] = u;
    ss = fmaf(u, u, ss);
  }
  const float norm = sqrtf(block_sum(ss, red));
  const float den = fmaxf(norm, IP_NORM_EPS);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = o[c] / den;
    o[c] = round ? tf32_round(v) : v;
  }
  if (threadIdx.x == 0) {
    ssum[(size_t)n * K + k] = s;
    nrm[(size_t)n * K + k] = norm;
  }
}

// Block (k, n): the adjoints of the normalisation and the residual coding.  du = (dout - o (o . dout)) / |u| (dout / 1e-12 in
// F.normalize's clamp); dq = du / (sigma S); ds = -sum_c du q / (sigma S^2), 0 where s < 1e-5 (the clamp); the direct centre
// gradient -du / sigma and dsigma = -sum_c du u / sigma, per image.
__global__ void ip_group_bwd_prep_kernel(const float* __restrict__ dout, const float* __restrict__ qx,
                                         const float* __restrict__ ssum, const float* __restrict__ nrm,
                                         const float* __restrict__ cen, const float* __restrict__ smooth,
                                         float* __restrict__ dq, float* __restrict__ dsum, float* __restrict__ dcd,
                                         float* __restrict__ dsig, int K, int C) {
  __shared__ float red[32];
  const int k = blockIdx.x, n = blockIdx.y;
  const size_t row = ((size_t)n * K + k) * C;
  const float s = ssum[(size_t)n * K + k], S = fmaxf(s, IP_SUM_EPS), sigma = sqrtf(ip_beta(smooth, k) / 2.f);
  const float norm = nrm[(size_t)n * K + k];
  const bool clamped = !(norm >= IP_NORM_EPS);
  const float den = clamped ? IP_NORM_EPS : norm;
  float od = 0.f;
  if (!clamped)
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const float u = (qx[row + c] / S - cen[(size_t)k * C + c]) / sigma;
      od = fmaf(u / den, dout[row + c], od);
    }
  od = block_sum(od, red);
  float dS = 0.f, dsg = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float q = qx[row + c];
    const float u = (q / S - cen[(size_t)k * C + c]) / sigma;
    const float du = clamped ? dout[row + c] / den : (dout[row + c] - (u / den) * od) / den;
    dq[row + c] = du / (sigma * S);
    dcd[row + c] = -du / sigma;
    dS = fmaf(du, q, dS);
    dsg = fmaf(du, u, dsg);
  }
  dS = block_sum(dS, red);
  dsg = block_sum(dsg, red);
  if (threadIdx.x == 0) {
    dsum[(size_t)n * K + k] = s >= IP_SUM_EPS ? -dS / (sigma * S * S) : 0.f;
    dsig[(size_t)n * K + k] = -dsg / sigma;
  }
}

// Block (tile t, image n).  One read of the tile, one write of its dx:
//   da[k, p] = dq_k . x_p + ds_k (+ dassign) (+ the shaping term: coef[n, k] w[tap] when p lies under the Gaussian window of
//   the blurred maximum argmax[n, k]); dz = a (da - sum_j a_j da_j); dD = -dz / beta; dbeta partial sum_p dz D / beta^2;
//   dx[p, :] = sum_k a dq_k + 2 dD (x_p - c_k); the tile's centre partial -2 sum_p dD (x_p - c_k).
__global__ void __launch_bounds__(256) ip_group_bwd_tile_kernel(
    const float* __restrict__ x, const float* __restrict__ cen, const float* __restrict__ smooth,
    const float* __restrict__ assign, const float* __restrict__ dist, const float* __restrict__ dq,
    const float* __restrict__ dsum, const float* __restrict__ dassign, const int* __restrict__ argmax,
    const float* __restrict__ coef, const float* __restrict__ gw, int radius, float* __restrict__ dx,
    float* __restrict__ pc, float* __restrict__ pb, int H, int W, int K, int C) {
  extern __shared__ float4 ip_smem[];
  float* xs = reinterpret_cast<float*>(ip_smem);
  float* as = xs + (size_t)IP_TP * C;                 // [K][IP_TP] assign
  float* gs = as + IP_MAX_K * IP_TP;                  // [K][IP_TP] da, then dD
  float* bs = gs + IP_MAX_K * IP_TP;                  // [K][IP_TP] dbeta terms
  const int HW = H * W;
  const int n = blockIdx.y, t = blockIdx.x, T = gridDim.x, p0 = t * IP_TP;
  const int valid = min(IP_TP, HW - p0);
  ip_load_tile(x, xs, n, p0, HW, C);
  for (int i = threadIdx.x; i < K * IP_TP; i += blockDim.x) {
    const int k = i / IP_TP, p = i % IP_TP;
    as[i] = p < valid ? assign[((size_t)n * K + k) * HW + p0 + p] : 0.f;
  }
  __syncthreads();
  ip_tile_pairs<true>(xs, dq + (size_t)n * K * C, gs, valid, K, C);
  __syncthreads();
  if (threadIdx.x < IP_TP) {
    const int p = threadIdx.x, pix = p0 + p;
    if (p < valid) {
      const int y = pix / W, xx = pix % W, S = 2 * radius + 1, Wo = W - 2 * radius;
      float ad = 0.f;
      for (int k = 0; k < K; ++k) {
        const size_t nk = (size_t)n * K + k;
        float da = gs[k * IP_TP + p] + dsum[nk];
        if (dassign) da += dassign[nk * HW + pix];
        if (coef) {
          const int am = argmax[nk], dy = y - am / Wo, dxx = xx - am % Wo;
          if (dy >= 0 && dy < S && dxx >= 0 && dxx < S) da = fmaf(coef[nk], gw[dy * S + dxx], da);
        }
        gs[k * IP_TP + p] = da;
        ad = fmaf(as[k * IP_TP + p], da, ad);
      }
      for (int k = 0; k < K; ++k) {
        const float beta = ip_beta(smooth, k);
        const float dz = as[k * IP_TP + p] * (gs[k * IP_TP + p] - ad);
        gs[k * IP_TP + p] = -dz / beta;
        bs[k * IP_TP + p] = dz * dist[((size_t)n * K + k) * HW + pix] / (beta * beta);
      }
    } else {
      for (int k = 0; k < K; ++k) gs[k * IP_TP + p] = bs[k * IP_TP + p] = 0.f;
    }
  }
  __syncthreads();
  const float* dqn = dq + (size_t)n * K * C;
  float* pct = pc + ((size_t)n * T + t) * K * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc[IP_TP];                                 // dx of the tile's pixels at channel c (rows past HW stay unused)
#pragma unroll
    for (int p = 0; p < IP_TP; ++p) acc[p] = 0.f;
    for (int k = 0; k < K; ++k) {
      const float dqk = dqn[(size_t)k * C + c], ck = cen[(size_t)k * C + c];
      float s = 0.f;
#pragma unroll
      for (int p = 0; p < IP_TP; ++p) {
        const float g = gs[k * IP_TP + p], d = xs[p * C + c] - ck;
        acc[p] = fmaf(as[k * IP_TP + p], dqk, fmaf(2.f * g, d, acc[p]));
        s = fmaf(g, d, s);
      }
      pct[(size_t)k * C + c] = -2.f * s;
    }
#pragma unroll
    for (int p = 0; p < IP_TP; ++p)
      if (p < valid) dx[((size_t)n * HW + p0 + p) * C + c] = acc[p];
  }
  if (threadIdx.x < K) {
    float s = 0.f;
    for (int p = 0; p < valid; ++p) s += bs[threadIdx.x * IP_TP + p];
    pb[((size_t)n * T + t) * K + threadIdx.x] = s;
  }
}

// Block per part k: dcen = sum_n (direct term) + sum_{n, t} (tile partials); dsmooth = (sum_n dsigma / (4 sigma) +
// sum_{n, t} dbeta partials) beta (1 - beta), all in ascending order.
__global__ void ip_group_bwd_finish_kernel(const float* __restrict__ dcd, const float* __restrict__ pc,
                                           const float* __restrict__ dsig, const float* __restrict__ pb,
                                           const float* __restrict__ smooth, float* __restrict__ dcen,
                                           float* __restrict__ dsmooth, int N, int T, int K, int C) {
  const int k = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    for (int n = 0; n < N; ++n) acc += dcd[((size_t)n * K + k) * C + c];
    for (int i = 0; i < N * T; ++i) acc += pc[((size_t)i * K + k) * C + c];
    dcen[(size_t)k * C + c] = acc;
  }
  if (threadIdx.x == 0) {
    const float beta = ip_beta(smooth, k), sigma = sqrtf(beta / 2.f);
    float ds = 0.f, db = 0.f;
    for (int n = 0; n < N; ++n) ds += dsig[(size_t)n * K + k];
    for (int i = 0; i < N * T; ++i) db += pb[(size_t)i * K + k];
    dsmooth[k] = (ds / (4.f * sigma) + db) * beta * (1.f - beta);
  }
}

// ---- part attention ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ip_att_pre(float c, float mean, float invstd, float gamma, float beta) {
  return (c - mean) * invstd * gamma + beta;
}

// One block.  conv[p] = f[p, :] . w + b (a warp per row); BatchNorm(1) over the P = N K values (train: batch mean and biased
// variance, running statistics updated with momentum and the unbiased variance; eval: the running statistics); ReLU; softmax
// over the K parts of each image.  stats = (mean, invstd) as used.
__global__ void ip_att_fwd_kernel(const float* __restrict__ f, const float* __restrict__ w, const float* __restrict__ b,
                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                  float* __restrict__ running_mean, float* __restrict__ running_var, float momentum,
                                  float eps, int training, float* __restrict__ conv, float* __restrict__ att,
                                  float* __restrict__ stats, int N, int K, int C) {
  __shared__ float red[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5, P = N * K;
  for (int p = warp; p < P; p += nw) {
    float acc = 0.f;
    for (int c = lane; c < C; c += 32) acc = fmaf(f[(size_t)p * C + c], w[c], acc);
    acc = warp_sum(acc);
    if (lane == 0) conv[p] = acc + b[0];
  }
  __syncthreads();
  float mean, invstd;
  if (training) {
    float s = 0.f;
    for (int p = threadIdx.x; p < P; p += blockDim.x) s += conv[p];
    mean = block_sum(s, red) / (float)P;
    float v = 0.f;
    for (int p = threadIdx.x; p < P; p += blockDim.x) v = fmaf(conv[p] - mean, conv[p] - mean, v);
    const float var = block_sum(v, red) / (float)P;
    invstd = rsqrtf(var + eps);
    if (threadIdx.x == 0) {
      running_mean[0] = (1.f - momentum) * running_mean[0] + momentum * mean;
      running_var[0] = (1.f - momentum) * running_var[0] + momentum * var * (float)P / (float)(P - 1);
    }
  } else {
    mean = running_mean[0];
    invstd = rsqrtf(running_var[0] + eps);
  }
  if (threadIdx.x == 0) {
    stats[0] = mean;
    stats[1] = invstd;
  }
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float m = -INFINITY;
    for (int k = 0; k < K; ++k) m = fmaxf(m, fmaxf(ip_att_pre(conv[n * K + k], mean, invstd, gamma[0], beta[0]), 0.f));
    float s = 0.f;
    for (int k = 0; k < K; ++k) s += expf(fmaxf(ip_att_pre(conv[n * K + k], mean, invstd, gamma[0], beta[0]), 0.f) - m);
    for (int k = 0; k < K; ++k)
      att[n * K + k] = expf(fmaxf(ip_att_pre(conv[n * K + k], mean, invstd, gamma[0], beta[0]), 0.f) - m) / s;
  }
}

// pooled[n, d] = sum_k att[n, k] post[n, k, d], ascending k.
__global__ void ip_att_pool_kernel(const float* __restrict__ att, const float* __restrict__ post, float* __restrict__ pooled,
                                   int K, int D) {
  const int n = blockIdx.y, d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(att[n * K + k], post[((size_t)n * K + k) * D + d], acc);
  pooled[(size_t)n * D + d] = acc;
}

// Block per row p = (n, k): datt[p] = dpooled[n] . post[p] (+ datt_in[p]); dpost[p, :] = att[p] dpooled[n, :].
__global__ void ip_att_bwd_pool_kernel(const float* __restrict__ att, const float* __restrict__ post,
                                       const float* __restrict__ dpooled, const float* __restrict__ datt_in,
                                       float* __restrict__ dpost, float* __restrict__ datt, int K, int D) {
  __shared__ float red[32];
  const int p = blockIdx.x, n = p / K;
  const float a = att[p];
  float acc = 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const float g = dpooled[(size_t)n * D + d];
    acc = fmaf(g, post[(size_t)p * D + d], acc);
    dpost[(size_t)p * D + d] = a * g;
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) datt[p] = datt_in ? acc + datt_in[p] : acc;
}

// One block: softmax adjoint per image, ReLU mask (the forward's expression re-evaluated), BatchNorm(1) adjoint (batch
// statistics in train mode, constants in eval mode) -> dconv [P] (in place of datt), dgamma, dbeta and the conv bias db.
__global__ void ip_att_bwd_bn_kernel(const float* __restrict__ conv, const float* __restrict__ att,
                                     const float* __restrict__ stats, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, float* __restrict__ g, float* __restrict__ db,
                                     float* __restrict__ dgamma, float* __restrict__ dbeta, int training, int N, int K) {
  __shared__ float red[32];
  const int P = N * K;
  const float mean = stats[0], invstd = stats[1], gm = gamma[0], bt = beta[0];
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float t = 0.f;
    for (int k = 0; k < K; ++k) t = fmaf(att[n * K + k], g[n * K + k], t);
    for (int k = 0; k < K; ++k) {
      const int p = n * K + k;
      const float dy = att[p] * (g[p] - t);
      g[p] = ip_att_pre(conv[p], mean, invstd, gm, bt) > 0.f ? dy : 0.f;
    }
  }
  __syncthreads();
  float sg = 0.f, sx = 0.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    sg += g[p];
    sx = fmaf(g[p], (conv[p] - mean) * invstd, sx);
  }
  sg = block_sum(sg, red);
  sx = block_sum(sx, red);
  float sc = 0.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const float xhat = (conv[p] - mean) * invstd;
    const float dc = training ? gm * invstd * (g[p] - sg / (float)P - xhat * sx / (float)P) : gm * invstd * g[p];
    g[p] = dc;
    sc += dc;
  }
  sc = block_sum(sc, red);
  if (threadIdx.x == 0) {
    dgamma[0] = sx;
    dbeta[0] = sg;
    db[0] = sc;
  }
}

// Thread per channel c: dw[c] = sum_p dconv[p] f[p, c] (ascending p); df[p, c] = dconv[p] w[c].
__global__ void ip_att_bwd_conv_kernel(const float* __restrict__ f, const float* __restrict__ w,
                                       const float* __restrict__ dconv, float* __restrict__ df, float* __restrict__ dw,
                                       int P, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float wc = w[c];
  float acc = 0.f;
  for (int p = 0; p < P; ++p) {
    const float g = dconv[p];
    acc = fmaf(g, f[(size_t)p * C + c], acc);
    df[(size_t)p * C + c] = g * wc;
  }
  dw[c] = acc;
}

// ---- shaping loss --------------------------------------------------------------------------------------------------------
// Block per (n, k): the "valid" Gaussian blur of assign[n, k] and its maximum; argmax = the first maximum in row-major
// order of the (H - 2r) x (W - 2r) blurred map.
__global__ void ip_occupancy_kernel(const float* __restrict__ assign, const float* __restrict__ gw, float* __restrict__ occ,
                                    int* __restrict__ argmax, int H, int W, int radius) {
  __shared__ float sb[32];
  __shared__ int si[32];
  const int S = 2 * radius + 1, Ho = H - 2 * radius, Wo = W - 2 * radius;
  const float* a = assign + (size_t)blockIdx.x * H * W;
  float best = -INFINITY;
  int arg = 0x7fffffff;
  for (int o = threadIdx.x; o < Ho * Wo; o += blockDim.x) {
    const int oy = o / Wo, ox = o % Wo;
    float v = 0.f;
    for (int i = 0; i < S; ++i)
      for (int j = 0; j < S; ++j) v = fmaf(gw[i * S + j], a[(oy + i) * W + ox + j], v);
    if (v > best) { best = v; arg = o; }
  }
  warp_argmax(best, arg);
  if ((threadIdx.x & 31) == 0) {
    sb[threadIdx.x >> 5] = best;
    si[threadIdx.x >> 5] = arg;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i)
      if (sb[i] > best || (sb[i] == best && si[i] < arg)) { best = sb[i]; arg = si[i]; }
    occ[blockIdx.x] = best;
    argmax[blockIdx.x] = arg;
  }
}

// One block.  Element (i, k) of occ [R, K] takes rank r = #{j : occ[j, k] < occ[i, k], or equal with j < i} in its column,
// i.e. its place in the ascending sort; term = log(occ + eps) - log(prior[r] + eps); loss = mean |term|;
// docc = sign(term) / ((occ + eps) R K), sign(0) = 0.
__global__ void ip_shaping_loss_kernel(const float* __restrict__ occ, const float* __restrict__ prior,
                                       float* __restrict__ loss, float* __restrict__ docc, int R, int K, float eps) {
  __shared__ float red[32];
  const float scale = 1.f / ((float)R * (float)K);
  float acc = 0.f;
  for (int e = threadIdx.x; e < R * K; e += blockDim.x) {
    const int i = e / K, k = e % K;
    const float v = occ[e];
    int r = 0;
    for (int j = 0; j < R; ++j) {
      const float o = occ[(size_t)j * K + k];
      r += (o < v) || (o == v && j < i);
    }
    const float term = logf(v + eps) - logf(prior[r] + eps);
    acc += fabsf(term);
    const float sg = term > 0.f ? 1.f : (term < 0.f ? -1.f : 0.f);
    docc[e] = sg / (v + eps) * scale;
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) loss[0] = acc * scale;
}

static int ip_check_group(int N, int HW, int K, int C, const char* op) {
  HK_REQUIRE(N > 0 && HW > 0 && K > 0 && C > 0, HK_ERR_ARG, "%s: N=%d HW=%d K=%d C=%d", op, N, HW, K, C);
  HK_REQUIRE(K <= IP_MAX_K, HK_ERR_UNSUPPORTED, "%s: K=%d parts above %d", op, K, IP_MAX_K);
  HK_REQUIRE(C % 4 == 0 && C <= IP_MAX_C, HK_ERR_UNSUPPORTED, "%s: C=%d must be a multiple of 4 and at most %d", op, C,
             IP_MAX_C);
  HK_REQUIRE(N <= 65535, HK_ERR_UNSUPPORTED, "%s: N=%d above 65535", op, N);
  return 0;
}

static int ip_tiles(int HW) { return (HW + IP_TP - 1) / IP_TP; }

static size_t ip_smem_bytes(int C) { return ((size_t)IP_TP * C + 3 * (size_t)IP_MAX_K * IP_TP) * sizeof(float); }

}  // namespace hk

using namespace hk;

extern "C" {

size_t hk_ip_group_workspace_bytes(int N, int HW, int K, int C) {
  const size_t T = (size_t)ip_tiles(HW > 0 ? HW : 1);
  const size_t nk = (size_t)N * K;
  // tile partials [N, T, K, C] + [N, T, K]; backward also dq and the direct centre term [N, K, C] and dsum, dsigma [N, K]
  return (nk * T * C + nk * T + 2 * nk * C + 2 * nk) * sizeof(float);
}

int hk_ip_group_fwd(const float* x, const float* centres, const float* smooth, float* assign, float* dist, float* out,
                    float* qx, float* ssum, float* nrm, int N, int HW, int K, int C, void* workspace,
                    size_t workspace_bytes, void* stream) {
  HK_REQUIRE(x && centres && smooth && assign && dist && out && qx && ssum && nrm && workspace, HK_ERR_ARG,
             "hk_ip_group_fwd: null pointer");
  if (int r = ip_check_group(N, HW, K, C, "hk_ip_group_fwd")) return r;
  HK_REQUIRE(aligned16(x) && aligned16(centres), HK_ERR_ALIGN, "hk_ip_group_fwd: x and centres must be 16-byte aligned");
  HK_REQUIRE(workspace_bytes >= hk_ip_group_workspace_bytes(N, HW, K, C), HK_ERR_WORKSPACE,
             "hk_ip_group_fwd: workspace %zu bytes, needs %zu", workspace_bytes, hk_ip_group_workspace_bytes(N, HW, K, C));
  const int T = ip_tiles(HW);
  float* pq = static_cast<float*>(workspace);
  float* ps = pq + (size_t)N * T * K * C;
  const size_t smem = ip_smem_bytes(C);
  if (int r = allow_dynamic_smem<ip_group_fwd_tile_kernel>((int)ip_smem_bytes(IP_MAX_C), "ip_group_fwd_tile_kernel"))
    return r;
  ip_group_fwd_tile_kernel<<<dim3(T, N), 256, smem, (cudaStream_t)stream>>>(x, centres, smooth, assign, dist, pq, ps, HW, K,
                                                                            C);
  HK_LAUNCH_CHECK("ip_group_fwd_tile_kernel");
  ip_group_fwd_finish_kernel<<<dim3(K, N), 256, 0, (cudaStream_t)stream>>>(pq, ps, centres, smooth, out, qx, ssum, nrm, T, K,
                                                                           C, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("ip_group_fwd_finish_kernel");
  return 0;
}

int hk_ip_group_bwd(const float* x, const float* centres, const float* smooth, const float* assign, const float* dist,
                    const float* qx, const float* ssum, const float* nrm, const float* dout, const float* dassign,
                    const int* argmax, const float* coef, const float* gauss, int radius, float* dx, float* dcentres,
                    float* dsmooth, int N, int H, int W, int K, int C, void* workspace, size_t workspace_bytes,
                    void* stream) {
  HK_REQUIRE(x && centres && smooth && assign && dist && qx && ssum && nrm && dout && dx && dcentres && dsmooth &&
                 workspace && (!coef || (argmax && gauss)),
             HK_ERR_ARG, "hk_ip_group_bwd: null pointer");
  HK_REQUIRE(H > 0 && W > 0, HK_ERR_ARG, "hk_ip_group_bwd: H=%d W=%d", H, W);
  const int HW = H * W;
  if (int r = ip_check_group(N, HW, K, C, "hk_ip_group_bwd")) return r;
  HK_REQUIRE(!coef || (radius >= 0 && 2 * radius < H && 2 * radius < W), HK_ERR_ARG,
             "hk_ip_group_bwd: radius=%d leaves no blurred output on a %dx%d map", radius, H, W);
  HK_REQUIRE(aligned16(x), HK_ERR_ALIGN, "hk_ip_group_bwd: x must be 16-byte aligned");
  HK_REQUIRE(workspace_bytes >= hk_ip_group_workspace_bytes(N, HW, K, C), HK_ERR_WORKSPACE,
             "hk_ip_group_bwd: workspace %zu bytes, needs %zu", workspace_bytes, hk_ip_group_workspace_bytes(N, HW, K, C));
  const int T = ip_tiles(HW);
  const size_t nk = (size_t)N * K;
  float* dq = static_cast<float*>(workspace);          // first: the tile kernel reads it as float4
  float* dcd = dq + nk * C;
  float* pc = dcd + nk * C;
  float* pb = pc + nk * T * C;
  float* dsum = pb + nk * T;
  float* dsig = dsum + nk;
  ip_group_bwd_prep_kernel<<<dim3(K, N), 256, 0, (cudaStream_t)stream>>>(dout, qx, ssum, nrm, centres, smooth, dq, dsum, dcd,
                                                                         dsig, K, C);
  HK_LAUNCH_CHECK("ip_group_bwd_prep_kernel");
  if (int r = allow_dynamic_smem<ip_group_bwd_tile_kernel>((int)ip_smem_bytes(IP_MAX_C), "ip_group_bwd_tile_kernel"))
    return r;
  ip_group_bwd_tile_kernel<<<dim3(T, N), 256, ip_smem_bytes(C), (cudaStream_t)stream>>>(
      x, centres, smooth, assign, dist, dq, dsum, dassign, argmax, coef, gauss, radius, dx, pc, pb, H, W, K, C);
  HK_LAUNCH_CHECK("ip_group_bwd_tile_kernel");
  ip_group_bwd_finish_kernel<<<K, 256, 0, (cudaStream_t)stream>>>(dcd, pc, dsig, pb, smooth, dcentres, dsmooth, N, T, K, C);
  HK_LAUNCH_CHECK("ip_group_bwd_finish_kernel");
  return 0;
}

int hk_ip_att_fwd(const float* f, const float* w, const float* b, const float* gamma, const float* beta,
                  float* running_mean, float* running_var, float momentum, float eps, int training, const float* post,
                  float* conv, float* att, float* stats, float* pooled, int N, int K, int C, int D, void* stream) {
  HK_REQUIRE(f && w && b && gamma && beta && running_mean && running_var && post && conv && att && stats && pooled,
             HK_ERR_ARG, "hk_ip_att_fwd: null pointer");
  HK_REQUIRE(N > 0 && K > 0 && C > 0 && D > 0, HK_ERR_ARG, "hk_ip_att_fwd: N=%d K=%d C=%d D=%d", N, K, C, D);
  HK_REQUIRE(!training || N * K > 1, HK_ERR_ARG,
             "hk_ip_att_fwd: BatchNorm in train mode needs more than one value (N=%d K=%d)", N, K);
  HK_REQUIRE(N <= 65535, HK_ERR_UNSUPPORTED, "hk_ip_att_fwd: N=%d above 65535", N);
  ip_att_fwd_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(f, w, b, gamma, beta, running_mean, running_var, momentum, eps,
                                                         training, conv, att, stats, N, K, C);
  HK_LAUNCH_CHECK("ip_att_fwd_kernel");
  ip_att_pool_kernel<<<dim3((D + 255) / 256, N), 256, 0, (cudaStream_t)stream>>>(att, post, pooled, K, D);
  HK_LAUNCH_CHECK("ip_att_pool_kernel");
  return 0;
}

int hk_ip_att_bwd(const float* f, const float* w, const float* gamma, const float* beta, const float* conv,
                  const float* att, const float* stats, const float* post, const float* dpooled, const float* datt,
                  int training, float* df,
                  float* dw, float* db, float* dgamma, float* dbeta, float* dpost, float* scratch, int N, int K, int C,
                  int D, void* stream) {
  HK_REQUIRE(f && w && gamma && beta && conv && att && stats && post && dpooled && df && dw && db && dgamma && dbeta &&
                 dpost && scratch,
             HK_ERR_ARG, "hk_ip_att_bwd: null pointer");
  HK_REQUIRE(N > 0 && K > 0 && C > 0 && D > 0, HK_ERR_ARG, "hk_ip_att_bwd: N=%d K=%d C=%d D=%d", N, K, C, D);
  const int P = N * K;
  ip_att_bwd_pool_kernel<<<P, 256, 0, (cudaStream_t)stream>>>(att, post, dpooled, datt, dpost, scratch, K, D);
  HK_LAUNCH_CHECK("ip_att_bwd_pool_kernel");
  ip_att_bwd_bn_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(conv, att, stats, gamma, beta, scratch, db, dgamma, dbeta,
                                                            training, N, K);
  HK_LAUNCH_CHECK("ip_att_bwd_bn_kernel");
  ip_att_bwd_conv_kernel<<<(C + 255) / 256, 256, 0, (cudaStream_t)stream>>>(f, w, scratch, df, dw, P, C);
  HK_LAUNCH_CHECK("ip_att_bwd_conv_kernel");
  return 0;
}

int hk_ip_occupancy(const float* assign, const float* gauss, float* occ, int* argmax, int N, int K, int H, int W,
                    int radius, void* stream) {
  HK_REQUIRE(assign && gauss && occ && argmax, HK_ERR_ARG, "hk_ip_occupancy: null pointer");
  HK_REQUIRE(N > 0 && K > 0 && H > 0 && W > 0 && radius >= 0, HK_ERR_ARG, "hk_ip_occupancy: N=%d K=%d H=%d W=%d radius=%d",
             N, K, H, W, radius);
  HK_REQUIRE(2 * radius < H && 2 * radius < W, HK_ERR_ARG,
             "hk_ip_occupancy: radius=%d leaves no blurred output on a %dx%d map", radius, H, W);
  ip_occupancy_kernel<<<N * K, 256, 0, (cudaStream_t)stream>>>(assign, gauss, occ, argmax, H, W, radius);
  HK_LAUNCH_CHECK("ip_occupancy_kernel");
  return 0;
}

int hk_ip_shaping_loss(const float* occ, const float* prior, float* loss, float* docc, int R, int K, float eps,
                       void* stream) {
  HK_REQUIRE(occ && prior && loss && docc, HK_ERR_ARG, "hk_ip_shaping_loss: null pointer");
  HK_REQUIRE(R > 0 && K > 0, HK_ERR_ARG, "hk_ip_shaping_loss: R=%d K=%d", R, K);
  ip_shaping_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(occ, prior, loss, docc, R, K, eps);
  HK_LAUNCH_CHECK("ip_shaping_loss_kernel");
  return 0;
}

}  // extern "C"
