// CrossX (reference model/methods/CrossX.py, model/loss/CrossX_loss.py): the multi-excitation residual of the MELayer
// blocks, the fusion of layer4 parts into layer3 parts with the global max of the layer3 part, and the loss (cross-entropy
// on the summed logits, the two KL terms and the three part-correlation regularisers) with its gradient, on the device.
//
// Part maps are laid out [N, HW, P, C] (the P parts of one pixel side by side): the spatial mean of all layer4 parts is one
// hk_apcnn_pool over [N, HW, P*C], which lands in the [N, P, C] layout the classifiers read.  Every sum runs in a fixed
// order (no atomics), so results are bitwise repeatable.
#include <math.h>

#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {
namespace {

constexpr int ME_SEG = 64;          // pixel rows per block of the excitation backward
constexpr int MAX_PARTS = 3;

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float& at(float4& v, int j) { return reinterpret_cast<float*>(&v)[j]; }
__device__ __forceinline__ float at(const float4& v, int j) { return reinterpret_cast<const float*>(&v)[j]; }
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }

// out = relu(c + r) (when out is given); part p = relu(c sigmoid(m[n, p]) + r), one float4 of channels per thread.
__global__ void me_fwd_kernel(const float* __restrict__ c, const float* __restrict__ r, const float* __restrict__ m,
                              float* __restrict__ out, float* __restrict__ parts, int N, int HW, int P, int C) {
  const int C4 = C / 4;
  const size_t total = (size_t)N * HW * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C4) * 4;
    const size_t pix = i / C4;
    const int n = (int)(pix / HW);
    const float4 cv = ld4(c + i * 4), rv = ld4(r + i * 4);
    if (out)
      st4(out + i * 4, make_float4(fmaxf(cv.x + rv.x, 0.f), fmaxf(cv.y + rv.y, 0.f), fmaxf(cv.z + rv.z, 0.f),
                                   fmaxf(cv.w + rv.w, 0.f)));
    for (int p = 0; p < P; ++p) {
      const float4 mv = ld4(m + ((size_t)n * P + p) * C + ch);
      st4(parts + (pix * P + p) * C + ch,
          make_float4(fmaxf(fmaf(cv.x, sigmoidf(mv.x), rv.x), 0.f), fmaxf(fmaf(cv.y, sigmoidf(mv.y), rv.y), 0.f),
                      fmaxf(fmaf(cv.z, sigmoidf(mv.z), rv.z), 0.f), fmaxf(fmaf(cv.w, sigmoidf(mv.w), rv.w), 0.f)));
    }
  }
}

// Block (segment s, 128 channels, image n): warp w takes the rows s*ME_SEG + w, + 8, ...; lane l the channels 4l..4l+3.
// dr = dout [c + r > 0] + sum_p dpart_p [part_p > 0], dc = dout [c + r > 0] + sum_p g_p dpart_p [part_p > 0], and the
// block's share of sum_hw dpart_p [part_p > 0] c goes to ws[s, n, p, :], the eight warps added in ascending order.
__global__ void __launch_bounds__(256) me_bwd_kernel(const float* __restrict__ c, const float* __restrict__ r,
                                                     const float* __restrict__ m, const float* __restrict__ dout,
                                                     const float* __restrict__ dparts, float* __restrict__ dc,
                                                     float* __restrict__ dr, float* __restrict__ ws, int N, int HW, int P,
                                                     int C) {
  __shared__ float4 red[8][MAX_PARTS][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int seg = blockIdx.x, n = blockIdx.z;
  const int ch = (blockIdx.y * 32 + lane) * 4;
  float4 g[MAX_PARTS], acc[MAX_PARTS];
#pragma unroll
  for (int p = 0; p < MAX_PARTS; ++p) {
    if (p >= P) break;
    const float4 mv = ld4(m + ((size_t)n * P + p) * C + ch);
    g[p] = make_float4(sigmoidf(mv.x), sigmoidf(mv.y), sigmoidf(mv.z), sigmoidf(mv.w));
    acc[p] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int end = min(HW, (seg + 1) * ME_SEG);
  for (int hw = seg * ME_SEG + warp; hw < end; hw += 8) {
    const size_t pix = (size_t)n * HW + hw, o = pix * C + ch;
    float4 cv = ld4(c + o), rv = ld4(r + o);
    float4 dcv = make_float4(0.f, 0.f, 0.f, 0.f), drv = dcv;
    if (dout) {
      const float4 dv = ld4(dout + o);
#pragma unroll
      for (int j = 0; j < 4; ++j) at(drv, j) = at(dcv, j) = at(cv, j) + at(rv, j) > 0.f ? at(dv, j) : 0.f;
    }
#pragma unroll
    for (int p = 0; p < MAX_PARTS; ++p) {
      if (p >= P) break;
      const float4 dp = ld4(dparts + (pix * P + p) * C + ch);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gj = at(g[p], j);
        const float d = fmaf(at(cv, j), gj, at(rv, j)) > 0.f ? at(dp, j) : 0.f;
        at(drv, j) += d;
        at(dcv, j) = fmaf(gj, d, at(dcv, j));
        at(acc[p], j) = fmaf(d, at(cv, j), at(acc[p], j));
      }
    }
    st4(dc + o, dcv);
    st4(dr + o, drv);
  }
#pragma unroll
  for (int p = 0; p < MAX_PARTS; ++p)
    if (p < P) red[warp][p][lane] = acc[p];
  __syncthreads();
  if (threadIdx.x < 32 * P) {
    const int p = threadIdx.x >> 5;
    float4 t = red[0][p][lane];
    for (int w = 1; w < 8; ++w) {
      const float4 v = red[w][p][lane];
      t = make_float4(t.x + v.x, t.y + v.y, t.z + v.z, t.w + v.w);
    }
    st4(ws + (((size_t)seg * N + n) * P + p) * C + ch, t);
  }
}

// dm[n, p, c] = g (1 - g) * sum over the segments, in ascending order, of ws[s, n, p, c].
__global__ void me_dm_kernel(const float* __restrict__ m, const float* __restrict__ ws, float* __restrict__ dm, int NPC,
                             int segs) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < NPC; i += gridDim.x * blockDim.x) {
    float t = 0.f;
    for (int s = 0; s < segs; ++s) t += ws[(size_t)s * NPC + i];
    const float g = sigmoidf(m[i]);
    dm[i] = g * (1.f - g) * t;
  }
}

// Block (32 channels, image n): thread (slot = tid / 8, q = tid % 8) takes the pixels slot, slot + 32, ... and the
// channels 4q..4q+3.  S = part_p + nearest-2x(R); the maximum of part_p over the pixels at the position ATen's adaptive max
// pool picks in its h-major scan (`val > max || isnan(val)`): the first of equal maxima, or the last NaN.
__global__ void __launch_bounds__(256) fuse_fwd_kernel(const float* __restrict__ parts, const float* __restrict__ R,
                                                       float* __restrict__ S, float* __restrict__ pmax,
                                                       int* __restrict__ pidx, int H, int W, int P, int C, int p) {
  __shared__ float sbest[32][33];
  __shared__ int sidx[32][33];
  const int q = threadIdx.x & 7, slot = threadIdx.x >> 3, n = blockIdx.y;
  const int ch = blockIdx.x * 32 + q * 4;
  const int HW = H * W, W2 = W / 2, H2 = H / 2;
  float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  int bi[4] = {0, 0, 0, 0};
  for (int hw = slot; hw < HW; hw += 32) {
    const int h = hw / W, w = hw - h * W;
    const size_t pix = (size_t)n * HW + hw;
    const float4 x = ld4(parts + (pix * P + p) * C + ch);
    const float4 rv = ld4(R + (((size_t)n * H2 + (h >> 1)) * W2 + (w >> 1)) * C + ch);
    st4(S + pix * C + ch, make_float4(x.x + rv.x, x.y + rv.y, x.z + rv.z, x.w + rv.w));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float v = at(x, j);
      if (v > at(best, j) || isnan(v)) { at(best, j) = v; bi[j] = hw; }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    sbest[slot][q * 4 + j] = at(best, j);
    sidx[slot][q * 4 + j] = bi[j];
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int k = threadIdx.x;
    float b = sbest[0][k];
    int i = sidx[0][k];
    for (int s = 1; s < 32; ++s) {
      const float v = sbest[s][k];
      const int vi = sidx[s][k];
      if (isnan(b)) {
        if (isnan(v) && vi > i) i = vi;
      } else if (isnan(v) || v > b || (v == b && vi < i)) {
        b = v;
        i = vi;
      }
    }
    const size_t o = ((size_t)n * P + p) * C + blockIdx.x * 32 + k;
    pmax[o] = b;
    pidx[o] = i;
  }
}

// One thread per (n, h2, w2, 4 channels) of R: dpart_p = dS + dmax at the max's pixel, dR = the 2x2 sum of dS.
__global__ void fuse_bwd_kernel(const float* __restrict__ dS, const float* __restrict__ dpmax, const int* __restrict__ pidx,
                                float* __restrict__ dparts, float* __restrict__ dR, int N, int H, int W, int P, int C, int p) {
  const int C4 = C / 4, H2 = H / 2, W2 = W / 2, HW = H * W;
  const size_t total = (size_t)N * H2 * W2 * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C4) * 4;
    const size_t cell = i / C4;
    const int w2 = (int)(cell % W2), h2 = (int)((cell / W2) % H2), n = (int)(cell / ((size_t)W2 * H2));
    const size_t po = ((size_t)n * P + p) * C + ch;
    const float4 dmx = ld4(dpmax + po);
    const int4 id = *reinterpret_cast<const int4*>(pidx + po);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int hw = (2 * h2 + (t >> 1)) * W + 2 * w2 + (t & 1);
      const size_t pix = (size_t)n * HW + hw;
      const float4 v = ld4(dS + pix * C + ch);
      acc = make_float4(acc.x + v.x, acc.y + v.y, acc.z + v.z, acc.w + v.w);
      st4(dparts + (pix * P + p) * C + ch, make_float4(v.x + (id.x == hw ? dmx.x : 0.f), v.y + (id.y == hw ? dmx.y : 0.f),
                                                       v.z + (id.z == hw ? dmx.z : 0.f), v.w + (id.w == hw ? dmx.w : 0.f)));
    }
    st4(dR + i * 4, acc);
  }
}

// 1 / ||x[0, C)|| by one warp, 0 for an all-zero row.
__device__ __forceinline__ float warp_inv_norm(const float* __restrict__ x, int C) {
  float ss = 0.f;
  for (int k = threadIdx.x & 31; k < C; k += 32) ss = fmaf(x[k], x[k], ss);
  ss = warp_sum(ss);
  return ss > 0.f ? 1.f / sqrtf(ss) : 0.f;
}

struct Feats {
  const float* f[3];
  int C[3];
  size_t off[3];    // offset of the group's [P, C] block in s
};

// Block (group g, part p): s[g][p][c] = sum_n x[n, p, c] / ||x[n, p]||, the images added in ascending order.
__global__ void reg_sums_kernel(Feats F, float* __restrict__ s, int N, int P) {
  extern __shared__ float inv[];
  const int g = blockIdx.x / P, p = blockIdx.x % P, C = F.C[g];
  const float* f = F.f[g];
  const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int n = warp; n < N; n += nw) {
    const float v = warp_inv_norm(f + ((size_t)n * P + p) * C, C);
    if ((threadIdx.x & 31) == 0) inv[n] = v;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < C; k += blockDim.x) {
    float t = 0.f;
    for (int n = 0; n < N; ++n) t = fmaf(f[((size_t)n * P + p) * C + k], inv[n], t);
    s[F.off[g] + (size_t)p * C + k] = t;
  }
}

// One block of 1024 threads.
//  * Warp per image: the label-smoothed cross-entropy of z = xf + xp + xc, KL(softmax xf || softmax xp) and
//    KL(softmax xf || softmax xc), each KL / N, and their gradients: dz = (softmax z - t) / N goes to all three logits,
//    dxp += (softmax xp - q) / N, dxc += (softmax xc - q) / N and dxf += q (a_p - KL_p + a_c - KL_c) / N with q = softmax xf,
//    a = log q - log softmax x (the target q is not detached).  The logit gradients are rounded to tf32 once (`round`).
//  * Group g (gamma_g, features [N, P, C_g]): corr[i, j] = s_i . s_j / n_total^2 and
//    L_g = gamma_g (sum_{i<j} corr[i, j] + sum_i (1 - corr[i, i])); dL/ds_i = gamma_g / n_total^2 (sum_j s_j - 3 s_i), and
//    a row's gradient is (ds - xhat (xhat . ds)) / ||x|| * reg_scale (0 for an all-zero row).
__global__ void __launch_bounds__(1024) crossx_loss_kernel(
    const float* __restrict__ xf, const float* __restrict__ xp, const float* __restrict__ xc,
    const long long* __restrict__ labels, Feats F, const float* __restrict__ s, float* __restrict__ loss,
    float* __restrict__ dxf, float* __restrict__ dxp, float* __restrict__ dxc, float* dfu, float* dfp, float* dfc,
    int* __restrict__ correct, int N, int K, int P, float eps, float gu, float gp, float gc, int n_total, float reg_scale,
    int round) {
  __shared__ float red[32];
  __shared__ int redi[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float invN = 1.f / (float)N;
  float ce = 0.f, kl = 0.f;
  int hits = 0;
  for (int n = warp; n < N; n += nw) {
    const size_t ro = (size_t)n * K;
    const float *f = xf + ro, *a = xp + ro, *b = xc + ro;
    float mz = -INFINITY, mf = -INFINITY, ma = -INFINITY, mb = -INFINITY;
    float best = -INFINITY;
    int am = 0;
    for (int k = lane; k < K; k += 32) {
      const float z = f[k] + a[k] + b[k];
      mz = fmaxf(mz, z);
      mf = fmaxf(mf, f[k]);
      ma = fmaxf(ma, a[k]);
      mb = fmaxf(mb, b[k]);
      if (z > best) { best = z; am = k; }
    }
    mz = warp_max(mz);
    mf = warp_max(mf);
    ma = warp_max(ma);
    mb = warp_max(mb);
    warp_argmax(best, am);
    float sz = 0.f, sl = 0.f, sf = 0.f, sa = 0.f, sb = 0.f;
    for (int k = lane; k < K; k += 32) {
      const float z = f[k] + a[k] + b[k];
      sz += expf(z - mz);
      sl += z;
      sf += expf(f[k] - mf);
      sa += expf(a[k] - ma);
      sb += expf(b[k] - mb);
    }
    const float lz = mz + logf(warp_sum(sz)), lf = mf + logf(warp_sum(sf));
    const float la = ma + logf(warp_sum(sa)), lb = mb + logf(warp_sum(sb));
    sl = warp_sum(sl);
    float ka = 0.f, kb = 0.f;
    for (int k = lane; k < K; k += 32) {
      const float lq = f[k] - lf, q = expf(lq);
      ka = fmaf(q, lq - (a[k] - la), ka);
      kb = fmaf(q, lq - (b[k] - lb), kb);
    }
    ka = warp_sum(ka);
    kb = warp_sum(kb);
    const long long y = labels[n];
    const bool valid = y >= 0 && y < K;
    const float zy = valid ? f[y] + a[y] + b[y] : lz;
    for (int k = lane; k < K; k += 32) {
      const float z = f[k] + a[k] + b[k];
      const float t = (k == y ? (1.f - eps) : 0.f) + eps / (float)K;
      const float gz = (expf(z - lz) - t) * invN;
      const float lq = f[k] - lf, q = expf(lq);
      const float pa = expf(a[k] - la), pb = expf(b[k] - lb);
      const float ga = gz + (pa - q) * invN, gb = gz + (pb - q) * invN;
      const float gf = gz + q * ((lq - (a[k] - la) - ka) + (lq - (b[k] - lb) - kb)) * invN;
      dxf[ro + k] = round ? tf32_round(gf) : gf;
      dxp[ro + k] = round ? tf32_round(ga) : ga;
      dxc[ro + k] = round ? tf32_round(gb) : gb;
    }
    if (lane == 0) {
      ce += fmaf(1.f - eps, lz - zy, eps * (lz - sl / (float)K));
      kl += ka + kb;
      hits += valid && am == y;
    }
  }
  const float t_ce = block_sum(ce, red);
  const float t_kl = block_sum(kl, red);
  const int t_hits = block_sum(hits, redi);

  const float gam[3] = {gu, gp, gc};
  float* dfs[3] = {dfu, dfp, dfc};
  const float inv_nt2 = 1.f / ((float)n_total * (float)n_total);
  float reg = 0.f;
  for (int g = 0; g < 3; ++g) {
    const int C = F.C[g];
    const float* sg = s + F.off[g];
    for (int i = 0; i < P; ++i)
      for (int j = i; j < P; ++j) {
        float d = 0.f;
        for (int k = threadIdx.x; k < C; k += blockDim.x) d = fmaf(sg[(size_t)i * C + k], sg[(size_t)j * C + k], d);
        d = block_sum(d, red) * inv_nt2;
        reg += gam[g] * (i == j ? 1.f - d : d);
      }
    const float coef = gam[g] * inv_nt2 * reg_scale;
    for (int row = warp; row < N * P; row += nw) {
      const int p = row % P;
      const float* x = F.f[g] + (size_t)row * C;
      float* dx = dfs[g] + (size_t)row * C;
      const float inv = warp_inv_norm(x, C);
      float dot = 0.f;
      for (int k = lane; k < C; k += 32) {
        float tot = 0.f;
        for (int j = 0; j < P; ++j) tot += sg[(size_t)j * C + k];
        dot = fmaf(x[k] * inv, fmaf(-3.f, sg[(size_t)p * C + k], tot), dot);
      }
      dot = warp_sum(dot);
      for (int k = lane; k < C; k += 32) {
        float tot = 0.f;
        for (int j = 0; j < P; ++j) tot += sg[(size_t)j * C + k];
        const float ds = fmaf(-3.f, sg[(size_t)p * C + k], tot);
        dx[k] = coef * inv * fmaf(-x[k] * inv, dot, ds);
      }
    }
  }
  if (threadIdx.x == 0) {
    loss[0] = t_ce * invN + t_kl * invN + reg;
    correct[0] = t_hits;
  }
}

Feats make_feats(const float* fu, const float* fp, const float* fc, int P, int Cu, int Cp) {
  Feats F;
  F.f[0] = fu;
  F.f[1] = fp;
  F.f[2] = fc;
  F.C[0] = Cu;
  F.C[1] = Cp;
  F.C[2] = Cp;
  F.off[0] = 0;
  F.off[1] = (size_t)P * Cu;
  F.off[2] = (size_t)P * (Cu + Cp);
  return F;
}

}  // namespace
}  // namespace hk

using namespace hk;

extern "C" {

int hk_crossx_me_fwd(const float* c, const float* r, const float* m, float* out, float* parts, int N, int HW, int P, int C,
                     void* stream) {
  HK_REQUIRE(c && r && m && parts, HK_ERR_ARG, "hk_crossx_me_fwd: null pointer");
  HK_REQUIRE(N > 0 && HW > 0 && P >= 1 && P <= 3 && C > 0 && C % 128 == 0, HK_ERR_ARG,
             "hk_crossx_me_fwd: N=%d HW=%d P=%d C=%d (P in 1..3, C %% 128)", N, HW, P, C);
  HK_REQUIRE(aligned16(c) && aligned16(r) && aligned16(m) && (!out || aligned16(out)) && aligned16(parts), HK_ERR_ALIGN,
             "hk_crossx_me_fwd: 16-byte alignment");
  me_fwd_kernel<<<grid_1d((size_t)N * HW * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(c, r, m, out, parts, N, HW, P, C);
  HK_LAUNCH_CHECK("me_fwd_kernel");
  return 0;
}

size_t hk_crossx_me_bwd_workspace_bytes(int N, int HW, int P, int C) {
  if (N <= 0 || HW <= 0 || P <= 0 || C <= 0) return 0;
  return (size_t)((HW + ME_SEG - 1) / ME_SEG) * N * P * C * sizeof(float);
}

int hk_crossx_me_bwd(const float* c, const float* r, const float* m, const float* dout, const float* dparts, float* dc,
                     float* dr, float* dm, int N, int HW, int P, int C, void* workspace, size_t workspace_bytes,
                     void* stream) {
  HK_REQUIRE(c && r && m && dparts && dc && dr && dm, HK_ERR_ARG, "hk_crossx_me_bwd: null pointer");
  HK_REQUIRE(N > 0 && N <= 65535 && HW > 0 && P >= 1 && P <= 3 && C > 0 && C % 128 == 0, HK_ERR_ARG,
             "hk_crossx_me_bwd: N=%d HW=%d P=%d C=%d (P in 1..3, C %% 128)", N, HW, P, C);
  HK_REQUIRE(workspace && workspace_bytes >= hk_crossx_me_bwd_workspace_bytes(N, HW, P, C), HK_ERR_WORKSPACE,
             "hk_crossx_me_bwd: workspace too small");
  HK_REQUIRE(aligned16(c) && aligned16(r) && aligned16(m) && (!dout || aligned16(dout)) && aligned16(dparts) &&
                 aligned16(dc) && aligned16(dr) && aligned16(workspace),
             HK_ERR_ALIGN, "hk_crossx_me_bwd: 16-byte alignment");
  const int segs = (HW + ME_SEG - 1) / ME_SEG;
  float* ws = static_cast<float*>(workspace);
  me_bwd_kernel<<<dim3(segs, C / 128, N), 256, 0, (cudaStream_t)stream>>>(c, r, m, dout, dparts, dc, dr, ws, N, HW, P, C);
  HK_LAUNCH_CHECK("me_bwd_kernel");
  const int npc = N * P * C;
  me_dm_kernel<<<grid_1d(npc, 256), 256, 0, (cudaStream_t)stream>>>(m, ws, dm, npc, segs);
  HK_LAUNCH_CHECK("me_dm_kernel");
  return 0;
}

int hk_crossx_fuse_fwd(const float* parts, const float* R, float* S, float* pmax, int* pidx, int N, int H, int W, int P,
                       int C, int p, void* stream) {
  HK_REQUIRE(parts && R && S && pmax && pidx, HK_ERR_ARG, "hk_crossx_fuse_fwd: null pointer");
  HK_REQUIRE(N > 0 && N <= 65535 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && P >= 1 && P <= 3 && p >= 0 && p < P &&
                 C > 0 && C % 32 == 0,
             HK_ERR_ARG, "hk_crossx_fuse_fwd: N=%d H=%d W=%d P=%d C=%d p=%d (H, W even, C %% 32, 0 <= p < P <= 3)", N, H, W,
             P, C, p);
  HK_REQUIRE(aligned16(parts) && aligned16(R) && aligned16(S), HK_ERR_ALIGN, "hk_crossx_fuse_fwd: 16-byte alignment");
  fuse_fwd_kernel<<<dim3(C / 32, N), 256, 0, (cudaStream_t)stream>>>(parts, R, S, pmax, pidx, H, W, P, C, p);
  HK_LAUNCH_CHECK("fuse_fwd_kernel");
  return 0;
}

int hk_crossx_fuse_bwd(const float* dS, const float* dpmax, const int* pidx, float* dparts, float* dR, int N, int H, int W,
                       int P, int C, int p, void* stream) {
  HK_REQUIRE(dS && dpmax && pidx && dparts && dR, HK_ERR_ARG, "hk_crossx_fuse_bwd: null pointer");
  HK_REQUIRE(N > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && P >= 1 && P <= 3 && p >= 0 && p < P && C > 0 &&
                 C % 4 == 0,
             HK_ERR_ARG, "hk_crossx_fuse_bwd: N=%d H=%d W=%d P=%d C=%d p=%d (H, W even, C %% 4, 0 <= p < P <= 3)", N, H, W,
             P, C, p);
  HK_REQUIRE(aligned16(dS) && aligned16(dpmax) && aligned16(pidx) && aligned16(dparts) && aligned16(dR), HK_ERR_ALIGN,
             "hk_crossx_fuse_bwd: 16-byte alignment");
  fuse_bwd_kernel<<<grid_1d((size_t)N * (H / 2) * (W / 2) * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(
      dS, dpmax, pidx, dparts, dR, N, H, W, P, C, p);
  HK_LAUNCH_CHECK("fuse_bwd_kernel");
  return 0;
}

int hk_crossx_reg_sums(const float* fu, const float* fp, const float* fc, float* s, int N, int P, int Cu, int Cp,
                       void* stream) {
  HK_REQUIRE(fu && fp && fc && s, HK_ERR_ARG, "hk_crossx_reg_sums: null pointer");
  HK_REQUIRE(N > 0 && N <= 8192 && P >= 1 && P <= 3 && Cu > 0 && Cp > 0, HK_ERR_ARG,
             "hk_crossx_reg_sums: N=%d P=%d Cu=%d Cp=%d (N <= 8192, P in 1..3)", N, P, Cu, Cp);
  reg_sums_kernel<<<3 * P, 256, N * sizeof(float), (cudaStream_t)stream>>>(make_feats(fu, fp, fc, P, Cu, Cp), s, N, P);
  HK_LAUNCH_CHECK("reg_sums_kernel");
  return 0;
}

int hk_crossx_loss(const float* xf, const float* xp, const float* xc, const long long* labels, const float* fu,
                   const float* fp, const float* fc, const float* s, float* loss, float* dxf, float* dxp, float* dxc,
                   float* dfu, float* dfp, float* dfc, int* correct, int N, int K, int P, int Cu, int Cp,
                   float label_smoothing, float gamma_ulti, float gamma_plty, float gamma_cmbn, int n_total,
                   float reg_scale, void* stream) {
  HK_REQUIRE(xf && xp && xc && labels && fu && fp && fc && s && loss && dxf && dxp && dxc && dfu && dfp && dfc && correct,
             HK_ERR_ARG, "hk_crossx_loss: null pointer");
  HK_REQUIRE(N > 0 && K > 0 && P >= 1 && P <= 3 && Cu > 0 && Cp > 0 && n_total >= N, HK_ERR_ARG,
             "hk_crossx_loss: N=%d K=%d P=%d Cu=%d Cp=%d n_total=%d (P in 1..3, n_total >= N)", N, K, P, Cu, Cp, n_total);
  crossx_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(xf, xp, xc, labels, make_feats(fu, fp, fc, P, Cu, Cp), s, loss,
                                                           dxf, dxp, dxc, dfu, dfp, dfc, correct, N, K, P, label_smoothing,
                                                           gamma_ulti, gamma_plty, gamma_cmbn, n_total, reg_scale,
                                                           precise() ? 0 : 1);
  HK_LAUNCH_CHECK("crossx_loss_kernel");
  return 0;
}

}  // extern "C"
