// Channel-interaction kernels (reference model/methods/CIN.py:24-60, ChannelInteractionModule): the row softmax of the
// negated channel Gram (:32), the contrastive weight |W_SCI - w * W_SCI_BA| (:51-53) and the spatial average pool of the
// classifier (:71-82).  The Gram, the W.X products, the 3x3 convolution and the fc layer run on the wgmma GEMM /
// implicit-GEMM kernels through the entry points of gemm.cu / conv.cu; these are the HBM-bound pieces in between.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

// w[r][:] = softmax(-g[r][:])   (one block per row)
__global__ void softmax_neg_rows_fwd_kernel(const float* __restrict__ g, float* __restrict__ w, int cols) {
  __shared__ float red[32];
  const float* gr = g + (size_t)blockIdx.x * cols;
  float* wr = w + (size_t)blockIdx.x * cols;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < cols; j += blockDim.x) m = fmaxf(m, -gr[j]);
  m = block_max(m, red);
  float s = 0.f;
  for (int j = threadIdx.x; j < cols; j += blockDim.x) s += expf(-gr[j] - m);
  const float inv = 1.f / block_sum(s, red);
  for (int j = threadIdx.x; j < cols; j += blockDim.x) wr[j] = expf(-gr[j] - m) * inv;
}
// dg = -(w * (dw - sum_j w_j dw_j))
__global__ void softmax_neg_rows_bwd_kernel(const float* __restrict__ w, const float* __restrict__ dw,
                                            float* __restrict__ dg, int cols) {
  __shared__ float red[32];
  const size_t off = (size_t)blockIdx.x * cols;
  float s = 0.f;
  for (int j = threadIdx.x; j < cols; j += blockDim.x) s = fmaf(w[off + j], dw[off + j], s);
  const float dot = block_sum(s, red);
  for (int j = threadIdx.x; j < cols; j += blockDim.x) dg[off + j] = -w[off + j] * (dw[off + j] - dot);
}

// w_cci[b] = | w_sci[b] - weight[b] * w_sci[(b + B/2) % B] |                                          (CIN.py:51-53)
__global__ void cci_weight_fwd_kernel(const float* __restrict__ w_sci, const float* __restrict__ weight,
                                      float* __restrict__ w_cci, int B, size_t per) {
  const size_t total = (size_t)B * per;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / per);
    const size_t e = i - (size_t)b * per;
    const int pb = (b + B / 2) % B;
    w_cci[i] = fabsf(w_sci[i] - weight[b] * w_sci[(size_t)pb * per + e]);
  }
}
// d_sci[x] = sign_x d[x] - weight[x'] sign_x' d[x'],  x' = (x + B/2) % B  (the sample whose partner x is);  gather form
// d_weight[b] = - sum_e sign_b d[b][e] w_sci[pb][e]   (d_weight pre-zeroed; block-reduced, one atomic per block)
__global__ void cci_weight_bwd_kernel(const float* __restrict__ w_sci, const float* __restrict__ weight,
                                      const float* __restrict__ d, float* __restrict__ d_sci, float* __restrict__ d_weight,
                                      int B, size_t per) {
  __shared__ float red[32];
  const int b = blockIdx.y;
  const int pb = (b + B / 2) % B;
  const float wb = weight[b], wpb = weight[pb];
  float acc = 0.f;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < per; e += (size_t)gridDim.x * blockDim.x) {
    const float a = w_sci[(size_t)b * per + e], p = w_sci[(size_t)pb * per + e];
    const float db_ = d[(size_t)b * per + e], dp = d[(size_t)pb * per + e];
    const float tb = a - wb * p;          // argument of |.| for sample b
    const float tp = p - wpb * a;         // argument of |.| for sample pb (whose partner is b, since (pb + B/2) % B == b)
    const float sb = tb > 0.f ? 1.f : (tb < 0.f ? -1.f : 0.f);
    const float sp = tp > 0.f ? 1.f : (tp < 0.f ? -1.f : 0.f);
    d_sci[(size_t)b * per + e] = sb * db_ - wpb * sp * dp;
    acc = fmaf(-sb * db_, p, acc);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) atomicAdd(d_weight + b, acc);
}

// y[r] = mean over the first `cols` entries of x[r][0..ld)          (AdaptiveAvgPool1d(1), CIN.py:71)
__global__ void row_mean_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long rows, int cols, int ld) {
  const long long r = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int j = lane; j < cols; j += 32) s += x[r * ld + j];
  s = warp_sum(s);
  if (lane == 0) y[r] = s / (float)cols;
}
__global__ void row_mean_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, long long rows, int cols, int ld) {
  const size_t total = (size_t)rows * ld;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const long long r = i / ld;
    const int j = (int)(i - r * ld);
    dx[i] = j < cols ? dy[r] / (float)cols : 0.f;
  }
}

// OSME excitation (reference model/methods/OSME.py:8-24): s[n][c][p] = sigmoid(m[n][c]) * x[n][c][p]
__global__ void se_gate_fwd_kernel(const float* __restrict__ x, const float* __restrict__ m, float* __restrict__ s,
                                   size_t rows, int hw) {
  const size_t total = rows * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const float g = 1.f / (1.f + expf(-m[i / hw]));
    s[i] = g * x[i];
  }
}
// dx = sigmoid(m) * ds ;  dm[n][c] = sigmoid'(m) * sum_p ds * x      (one warp per (n, c) row)
__global__ void se_gate_bwd_kernel(const float* __restrict__ x, const float* __restrict__ m, const float* __restrict__ ds,
                                   float* __restrict__ dx, float* __restrict__ dm, long long rows, int hw) {
  const long long r = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const float g = 1.f / (1.f + expf(-m[r]));
  float acc = 0.f;
  for (int p = lane; p < hw; p += 32) {
    const float d = ds[r * hw + p];
    acc = fmaf(d, x[r * hw + p], acc);
    dx[r * hw + p] = g * d;
  }
  acc = warp_sum(acc);
  if (lane == 0) dm[r] = acc * g * (1.f - g);
}

// CIN's contrastive loss (reference model/loss/CIN_loss.py:26-46).  d[i] = z[i] - z[half + i] over the flattened
// [B, F] map: the pairs' difference before the projection h, whose bias cancels in h(a) - h(b).  Rounded to tf32 when
// `round` (the default mode), as every operand handed to a single-pass TF32 product is.
__global__ void cin_pair_diff_fwd_kernel(const float* __restrict__ z, float* __restrict__ d, size_t n, int round) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = z[i] - z[n + i];
    d[i] = round ? tf32_round(v) : v;
  }
}
// dz = [dd; -dd]
__global__ void cin_pair_diff_bwd_kernel(const float* __restrict__ dd, float* __restrict__ dz, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float g = dd[i];
    dz[i] = g;
    dz[n + i] = -g;
  }
}

// nn.PairwiseDistance's eps: ||a - b + eps|| (CIN_loss.py:19)
constexpr float kPairwiseEps = 1e-6f;

// One block.  Pair i (< B/2) is matched when labels[i] == labels[B/2] (CIN_loss.py:39: every label of the first half
// against the single label labels[B/2]).  L1 = sum over matched i of ||p_i + eps||^2; the hinge term of :40-42 is
// overwritten by L1^2 at :43, so loss = alpha (L1 + L1^2) and dp_i = alpha (1 + 2 L1) 2 (p_i + eps) on matched rows, 0 on
// the others.  The sum runs in fp32 in a fixed order, so the result has the same bits on every run.
__global__ void cin_contrastive_loss_kernel(const float* __restrict__ p, const long long* __restrict__ labels,
                                            float* __restrict__ loss, float* __restrict__ dp, int B, int R, float alpha) {
  __shared__ float red[32];
  const int half = B / 2;
  const long long anchor = labels[half];
  const size_t n = (size_t)half * R;
  float s = 0.f;
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
    if (labels[i / R] != anchor) continue;
    const float v = p[i] + kPairwiseEps;
    s = fmaf(v, v, s);
  }
  const float l1 = block_sum(s, red);
  const float scale = 2.f * alpha * fmaf(2.f, l1, 1.f);
  for (size_t i = threadIdx.x; i < n; i += blockDim.x)
    dp[i] = labels[i / R] == anchor ? scale * (p[i] + kPairwiseEps) : 0.f;
  if (threadIdx.x == 0) loss[0] = alpha * fmaf(l1, l1, l1);
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_softmax_neg_rows_fwd(const float* g, float* w, long long rows, int cols, void* stream) {
  HK_REQUIRE(g && w && rows > 0 && cols > 0 && rows < (1ll << 31), HK_ERR_ARG, "hk_softmax_neg_rows_fwd: bad args");
  softmax_neg_rows_fwd_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(g, w, cols);
  HK_LAUNCH_CHECK("softmax_neg_rows_fwd_kernel");
  return 0;
}
int hk_softmax_neg_rows_bwd(const float* w, const float* dw, float* dg, long long rows, int cols, void* stream) {
  HK_REQUIRE(w && dw && dg && rows > 0 && cols > 0 && rows < (1ll << 31), HK_ERR_ARG, "hk_softmax_neg_rows_bwd: bad args");
  softmax_neg_rows_bwd_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(w, dw, dg, cols);
  HK_LAUNCH_CHECK("softmax_neg_rows_bwd_kernel");
  return 0;
}
int hk_cci_weight_fwd(const float* w_sci, const float* weight, float* w_cci, int B, long long per, void* stream) {
  HK_REQUIRE(w_sci && weight && w_cci && B > 0 && B % 2 == 0 && per > 0, HK_ERR_ARG, "hk_cci_weight_fwd: bad args (B must be even)");
  cci_weight_fwd_kernel<<<grid_1d((size_t)B * per, 256), 256, 0, (cudaStream_t)stream>>>(w_sci, weight, w_cci, B, (size_t)per);
  HK_LAUNCH_CHECK("cci_weight_fwd_kernel");
  return 0;
}
int hk_cci_weight_bwd(const float* w_sci, const float* weight, const float* d_cci, float* d_sci, float* d_weight, int B,
                      long long per, void* stream) {
  HK_REQUIRE(w_sci && weight && d_cci && d_sci && d_weight && B > 0 && B % 2 == 0 && per > 0, HK_ERR_ARG,
             "hk_cci_weight_bwd: bad args (B must be even)");
  cudaError_t e = cudaMemsetAsync(d_weight, 0, (size_t)B * sizeof(float), (cudaStream_t)stream);
  if (e != cudaSuccess) return set_error((int)e, "cudaMemsetAsync(d_weight): %s", cudaGetErrorString(e));
  cci_weight_bwd_kernel<<<dim3(64, B), 256, 0, (cudaStream_t)stream>>>(w_sci, weight, d_cci, d_sci, d_weight, B, (size_t)per);
  HK_LAUNCH_CHECK("cci_weight_bwd_kernel");
  return 0;
}
int hk_cin_pair_diff_fwd(const float* z, float* d, int B, long long per, void* stream) {
  HK_REQUIRE(z && d && B > 0 && B % 2 == 0 && per > 0, HK_ERR_ARG, "hk_cin_pair_diff_fwd: bad args (B must be even)");
  const size_t n = (size_t)(B / 2) * per;
  cin_pair_diff_fwd_kernel<<<grid_1d(n, 256), 256, 0, (cudaStream_t)stream>>>(z, d, n, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("cin_pair_diff_fwd_kernel");
  return 0;
}
int hk_cin_pair_diff_bwd(const float* dd, float* dz, int B, long long per, void* stream) {
  HK_REQUIRE(dd && dz && B > 0 && B % 2 == 0 && per > 0, HK_ERR_ARG, "hk_cin_pair_diff_bwd: bad args (B must be even)");
  const size_t n = (size_t)(B / 2) * per;
  cin_pair_diff_bwd_kernel<<<grid_1d(n, 256), 256, 0, (cudaStream_t)stream>>>(dd, dz, n);
  HK_LAUNCH_CHECK("cin_pair_diff_bwd_kernel");
  return 0;
}
int hk_cin_contrastive_loss(const float* p, const long long* labels, float* loss, float* dp, int B, int R, float alpha,
                            void* stream) {
  HK_REQUIRE(p && labels && loss && dp, HK_ERR_ARG, "hk_cin_contrastive_loss: null pointer");
  HK_REQUIRE(B > 0 && B % 2 == 0 && R > 0, HK_ERR_ARG, "hk_cin_contrastive_loss: B=%d must be even and positive, R=%d > 0",
             B, R);
  cin_contrastive_loss_kernel<<<1, 512, 0, (cudaStream_t)stream>>>(p, labels, loss, dp, B, R, alpha);
  HK_LAUNCH_CHECK("cin_contrastive_loss_kernel");
  return 0;
}
int hk_se_gate_fwd(const float* x, const float* m, float* s, long long rows, int hw, void* stream) {
  HK_REQUIRE(x && m && s && rows > 0 && hw > 0, HK_ERR_ARG, "hk_se_gate_fwd: bad args");
  se_gate_fwd_kernel<<<grid_1d((size_t)rows * hw, 256), 256, 0, (cudaStream_t)stream>>>(x, m, s, (size_t)rows, hw);
  HK_LAUNCH_CHECK("se_gate_fwd_kernel");
  return 0;
}
int hk_se_gate_bwd(const float* x, const float* m, const float* ds, float* dx, float* dm, long long rows, int hw,
                   void* stream) {
  HK_REQUIRE(x && m && ds && dx && dm && rows > 0 && hw > 0, HK_ERR_ARG, "hk_se_gate_bwd: bad args");
  se_gate_bwd_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, m, ds, dx, dm, rows, hw);
  HK_LAUNCH_CHECK("se_gate_bwd_kernel");
  return 0;
}
int hk_row_mean_fwd(const float* x, float* y, long long rows, int cols, int ld, void* stream) {
  HK_REQUIRE(x && y && rows > 0 && cols > 0 && ld >= cols, HK_ERR_ARG, "hk_row_mean_fwd: bad args");
  row_mean_fwd_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, y, rows, cols, ld);
  HK_LAUNCH_CHECK("row_mean_fwd_kernel");
  return 0;
}
int hk_row_mean_bwd(const float* dy, float* dx, long long rows, int cols, int ld, void* stream) {
  HK_REQUIRE(dy && dx && rows > 0 && cols > 0 && ld >= cols, HK_ERR_ARG, "hk_row_mean_bwd: bad args");
  row_mean_bwd_kernel<<<grid_1d((size_t)rows * ld, 256), 256, 0, (cudaStream_t)stream>>>(dy, dx, rows, cols, ld);
  HK_LAUNCH_CHECK("row_mean_bwd_kernel");
  return 0;
}

}  // extern "C"
