// Destruction and construction learning (reference model/methods/DCL.py, model/loss/DCL_loss.py): the region-alignment
// head (global average pool + 1x1 Convmask + AvgPool2d(2) + tanh, DCL.py:31-39) forward and backward, each one pass over
// the trunk map plus a small fixed-order finish, and the loss (two label-smoothed cross-entropies + an L1 term,
// DCL_loss.py:16-21) with its gradient in one launch.  The two bias-free classifiers run on hk_linear_*.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

constexpr int DCL_WARPS = 8;              // warps per head block
constexpr int DCL_CHUNK = 64;             // channels per head block (8 per warp)
constexpr int DCL_MAX_HW = 1024;          // per-warp z rows in shared memory: 8 x 1024 floats = 32 KB

static int dcl_chunks(int C) { return (C + DCL_CHUNK - 1) / DCL_CHUNK; }

// Block (chunk k, image n): warp w takes channels c0 + w, c0 + w + 8, ... of the chunk and reads each row x[n, c, :] once:
// its lane-strided sum gives pooled[n, c], and w[c] x[n, c, p] accumulates into the warp's own z row in shared memory (each
// position p is owned by one lane, so no synchronisation inside the loop).  The eight warp rows are then added in warp order
// into zpart[n, k, :]: the chunk's share of the Convmask output before the bias.
__global__ void dcl_head_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ pooled,
                                    float* __restrict__ zpart, int C, int HW, int round) {
  extern __shared__ float zs[];
  const int k = blockIdx.x, n = blockIdx.y, chunks = gridDim.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* zw = zs + warp * HW;
  for (int p = lane; p < HW; p += 32) zw[p] = 0.f;
  const int c1 = min(C, (k + 1) * DCL_CHUNK);
  for (int c = k * DCL_CHUNK + warp; c < c1; c += DCL_WARPS) {
    const float* row = x + ((size_t)n * C + c) * HW;
    const float wc = w[c];
    float s = 0.f;
    for (int p = lane; p < HW; p += 32) {
      const float v = row[p];
      s += v;
      zw[p] = fmaf(wc, v, zw[p]);
    }
    s = warp_sum(s);
    if (lane == 0) {
      const float m = s / (float)HW;
      pooled[(size_t)n * C + c] = round ? tf32_round(m) : m;     // operand of the classifier MMA
    }
  }
  __syncthreads();
  float* out = zpart + ((size_t)n * chunks + k) * HW;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < DCL_WARPS; ++i) t += zs[i * HW + p];
    out[p] = t;
  }
}

// mask[n, q] = tanh(mean of the 2x2 window q of z), z[p] = b + sum over chunks of zpart (ascending chunk order).  Windows
// tile the map from the top-left corner; an odd last row / column belongs to no window, as in AvgPool2d(2).
__global__ void dcl_head_finish_kernel(const float* __restrict__ zpart, const float* __restrict__ b, float* __restrict__ mask,
                                       int N, int H, int W, int chunks) {
  const int Ho = H / 2, Wo = W / 2, Q = Ho * Wo, HW = H * W;
  const float bias = b[0];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N * Q; i += gridDim.x * blockDim.x) {
    const int n = i / Q, q = i - n * Q;
    const int p = (q / Wo) * 2 * W + (q % Wo) * 2;
    const float* zp = zpart + (size_t)n * chunks * HW;
    float z00 = 0.f, z01 = 0.f, z10 = 0.f, z11 = 0.f;
    for (int k = 0; k < chunks; ++k, zp += HW) {
      z00 += zp[p];
      z01 += zp[p + 1];
      z10 += zp[p + W];
      z11 += zp[p + W + 1];
    }
    mask[i] = tanhf((((z00 + bias) + (z01 + bias)) + ((z10 + bias) + (z11 + bias))) * 0.25f);
  }
}

// Block (chunk k, image n): dz[p] = dmask[q] (1 - mask[q]^2) / 4 for p in window q, 0 off the windows, into shared memory;
// then each warp streams its channels: dx[n, c, p] = dpooled[n, c] / HW + w[c] dz[p] (one read of x, one write of dx) and
// dwpart[n, c] = sum_p x[n, c, p] dz[p] (lane-strided, then the fixed xor tree).
__global__ void dcl_head_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ mask,
                                    const float* __restrict__ dpooled, const float* __restrict__ dmask, float* __restrict__ dx,
                                    float* __restrict__ dwpart, int C, int H, int W) {
  extern __shared__ float dz[];
  const int k = blockIdx.x, n = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int HW = H * W, Ho = H / 2, Wo = W / 2, Q = Ho * Wo;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const int qy = (p / W) >> 1, qx = (p % W) >> 1;
    float g = 0.f;
    if (qy < Ho && qx < Wo) {
      const int q = n * Q + qy * Wo + qx;
      const float m = mask[q];
      g = dmask[q] * (1.f - m * m) * 0.25f;
    }
    dz[p] = g;
  }
  __syncthreads();
  const int c1 = min(C, (k + 1) * DCL_CHUNK);
  for (int c = k * DCL_CHUNK + warp; c < c1; c += DCL_WARPS) {
    const size_t off = ((size_t)n * C + c) * HW;
    const float dp = dpooled[(size_t)n * C + c] / (float)HW, wc = w[c];
    float acc = 0.f;
    for (int p = lane; p < HW; p += 32) {
      const float g = dz[p];
      acc = fmaf(x[off + p], g, acc);
      dx[off + p] = fmaf(wc, g, dp);
    }
    acc = warp_sum(acc);
    if (lane == 0) dwpart[(size_t)n * C + c] = acc;
  }
}

// dw[c] = sum_n dwpart[n, c] in ascending n; block 0's first warp also forms db = sum_{n,q} dmask (1 - mask^2) (each window
// passes a quarter of its gradient to four positions) lane-strided, then the fixed xor tree.
__global__ void dcl_head_bwd_finish_kernel(const float* __restrict__ dwpart, const float* __restrict__ mask,
                                           const float* __restrict__ dmask, float* __restrict__ dw, float* __restrict__ db,
                                           int N, int C, int NQ) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    float t = 0.f;
    for (int n = 0; n < N; ++n) t += dwpart[(size_t)n * C + c];
    dw[c] = t;
  }
  if (blockIdx.x == 0 && threadIdx.x < 32) {
    float t = 0.f;
    for (int i = threadIdx.x; i < NQ; i += 32) {
      const float m = mask[i];
      t = fmaf(dmask[i], 1.f - m * m, t);
    }
    t = warp_sum(t);
    if (threadIdx.x == 0) db[0] = t;
  }
}

// One block; warp w takes rows w, w + 32, ...  Per row: CE_ls(z[0, K), y), CE_ls(z[K, K + K2), y_swap), the gradient of
// both (pad columns [K + K2, ld) zeroed), the L1 term over the Q mask entries with d|m - l| = sign(m - l) (0 at equality),
// and the top-1 hit over z[0, K) or, with `combine` (cls_2xmul), over z[k] + z[K + k] + z[2K + k].  The per-warp fp64 sums
// are folded in warp order, so the loss is the same on every run.
__global__ void dcl_loss_kernel(const float* __restrict__ logits, int ld, int K, int K2, const long long* __restrict__ labels,
                                const long long* __restrict__ labels_swap, const float* __restrict__ mask,
                                const float* __restrict__ law, int R, int Q, float alpha, float beta, float gamma, int combine,
                                double* __restrict__ loss_acc, float* __restrict__ dlogits, float* __restrict__ dmask,
                                int* __restrict__ correct, int round) {
  __shared__ double red[32];
  __shared__ int s_corr[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const float eps = 0.1f;
  const float ls = gamma / ((float)R * (float)Q);
  double ce = 0.0, sw = 0.0, l1 = 0.0;
  int hits = 0;
  for (int r = warp; r < R; r += nw) {
    const float* z = logits + (size_t)r * ld;
    float* g = dlogits + (size_t)r * ld;
    const long long y = labels[r];
    const float c1 = warp_ce_ls(z, K, y, eps, alpha / (float)R, g, round);
    const float c2 = warp_ce_ls(z + K, K2, labels_swap[r], eps, beta / (float)R, g + K, round);
    for (int k = K + K2 + lane; k < ld; k += 32) g[k] = 0.f;
    float best = -INFINITY;
    int am = 0;
    for (int k = lane; k < K; k += 32) {
      const float v = combine ? (z[k] + z[K + k]) + z[2 * K + k] : z[k];
      if (v > best) { best = v; am = k; }
    }
    warp_argmax(best, am);
    const float* mr = mask + (size_t)r * Q;
    const float* lr = law + (size_t)r * Q;
    float a = 0.f;
    for (int q = lane; q < Q; q += 32) {
      const float d = mr[q] - lr[q];
      a += fabsf(d);
      dmask[(size_t)r * Q + q] = d > 0.f ? ls : (d < 0.f ? -ls : 0.f);
    }
    a = warp_sum(a);
    if (lane == 0) {
      ce += (double)c1;
      sw += (double)c2;
      l1 += (double)a;
      hits += (am == y);
    }
  }
  // ce, sw, l1, hits are 0 outside lane 0
  const double a = block_sum(ce, red), b = block_sum(sw, red), c = block_sum(l1, red);
  const int h = block_sum(hits, s_corr);
  if (threadIdx.x == 0) {
    loss_acc[0] += (double)alpha * (a / R) + (double)beta * (b / R) + (double)gamma * (c / ((double)R * Q));
    if (correct) correct[0] = h;
  }
}

static int check_head(int N, int C, int H, int W, const char* op) {
  HK_REQUIRE(N > 0 && C > 0 && H >= 2 && W >= 2, HK_ERR_ARG, "%s: N=%d C=%d H=%d W=%d (H, W >= 2)", op, N, C, H, W);
  HK_REQUIRE(H * W <= DCL_MAX_HW, HK_ERR_UNSUPPORTED, "%s: H*W=%d above %d", op, H * W, DCL_MAX_HW);
  return 0;
}

}  // namespace hk

using namespace hk;

extern "C" {

size_t hk_dcl_head_workspace_bytes(int N, int C, int H, int W) {
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0) return 0;
  const size_t fwd = (size_t)N * dcl_chunks(C) * H * W, bwd = (size_t)N * C;
  return (fwd > bwd ? fwd : bwd) * sizeof(float);
}

int hk_dcl_head_fwd(const float* x, const float* w, const float* b, float* pooled, float* mask, int N, int C, int H, int W,
                    void* workspace, size_t workspace_bytes, void* stream) {
  HK_REQUIRE(x && w && b && pooled && mask && workspace, HK_ERR_ARG, "hk_dcl_head_fwd: null pointer");
  if (int r = check_head(N, C, H, W, "hk_dcl_head_fwd")) return r;
  HK_REQUIRE(workspace_bytes >= hk_dcl_head_workspace_bytes(N, C, H, W), HK_ERR_WORKSPACE,
             "hk_dcl_head_fwd: workspace too small");
  const int chunks = dcl_chunks(C), HW = H * W;
  float* zpart = static_cast<float*>(workspace);
  dcl_head_fwd_kernel<<<dim3(chunks, N), DCL_WARPS * 32, DCL_WARPS * HW * sizeof(float), (cudaStream_t)stream>>>(
      x, w, pooled, zpart, C, HW, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("dcl_head_fwd_kernel");
  dcl_head_finish_kernel<<<grid_1d((size_t)N * (H / 2) * (W / 2), 256), 256, 0, (cudaStream_t)stream>>>(zpart, b, mask, N, H,
                                                                                                         W, chunks);
  HK_LAUNCH_CHECK("dcl_head_finish_kernel");
  return 0;
}

int hk_dcl_head_bwd(const float* x, const float* w, const float* mask, const float* dpooled, const float* dmask, float* dx,
                    float* dw, float* db, int N, int C, int H, int W, void* workspace, size_t workspace_bytes,
                    void* stream) {
  HK_REQUIRE(x && w && mask && dpooled && dmask && dx && dw && db && workspace, HK_ERR_ARG,
             "hk_dcl_head_bwd: null pointer");
  if (int r = check_head(N, C, H, W, "hk_dcl_head_bwd")) return r;
  HK_REQUIRE(workspace_bytes >= hk_dcl_head_workspace_bytes(N, C, H, W), HK_ERR_WORKSPACE,
             "hk_dcl_head_bwd: workspace too small");
  float* dwpart = static_cast<float*>(workspace);
  dcl_head_bwd_kernel<<<dim3(dcl_chunks(C), N), DCL_WARPS * 32, H * W * sizeof(float), (cudaStream_t)stream>>>(
      x, w, mask, dpooled, dmask, dx, dwpart, C, H, W);
  HK_LAUNCH_CHECK("dcl_head_bwd_kernel");
  dcl_head_bwd_finish_kernel<<<grid_1d(C, 256), 256, 0, (cudaStream_t)stream>>>(dwpart, mask, dmask, dw, db, N, C,
                                                                                N * (H / 2) * (W / 2));
  HK_LAUNCH_CHECK("dcl_head_bwd_finish_kernel");
  return 0;
}

int hk_dcl_loss(const float* logits, int ld, int K, int K2, const long long* labels, const long long* labels_swap,
                const float* mask, const float* law, int R, int Q, float alpha, float beta, float gamma, int combine,
                double* loss_acc, float* dlogits, float* dmask, int* correct, void* stream) {
  HK_REQUIRE(logits && labels && labels_swap && mask && law && loss_acc && dlogits && dmask, HK_ERR_ARG,
             "hk_dcl_loss: null pointer");
  HK_REQUIRE(R > 0 && Q > 0 && K > 0 && K2 > 0 && K + K2 <= ld, HK_ERR_ARG, "hk_dcl_loss: R=%d Q=%d K=%d K2=%d ld=%d", R, Q,
             K, K2, ld);
  HK_REQUIRE(!combine || K2 == 2 * K, HK_ERR_ARG, "hk_dcl_loss: combine needs K2 == 2K (K=%d, K2=%d)", K, K2);
  dcl_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(logits, ld, K, K2, labels, labels_swap, mask, law, R, Q, alpha, beta,
                                                        gamma, combine, loss_acc, dlogits, dmask, correct,
                                                        precise() ? 0 : 1);
  HK_LAUNCH_CHECK("dcl_loss_kernel");
  return 0;
}

}  // extern "C"
