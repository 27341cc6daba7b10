// Classifier head glue, loss and optimizer kernels of the training step (reference train.py:310-320):
//   * the skinny classifier GEMMs (nn.Linear(512**2, K), BCNN.py:42), split-K in the forward
//   * CrossEntropyLoss(label_smoothing=0.1) forward+backward (train.py:211-212), mean reduction
//   * fused SGD-momentum / Adam parameter update over flat fp32 buffers (Examples/BCNN.py:40, Examples/MPN.py:14-18)
#include "common.cuh"
#include "host.h"
#include "gemm.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

// One block; warps stride over rows.  loss = mean_b [ (1-eps) * -logp[y] + eps/K * sum_k -logp[k] ]
// dlogits = (softmax - ((1-eps) onehot + eps/K)) * grad_scale / B, rounded in tf32 mode: the operand of the classifier
// dgrad / wgrad MMAs.
__global__ void softmax_ce_ls_kernel(const float* __restrict__ logits, const long long* __restrict__ labels,
                                     float* __restrict__ loss, float* __restrict__ dlogits, int* __restrict__ correct,
                                     int B, int K, float eps, float grad_scale, int round) {
  __shared__ float s_loss[32];
  __shared__ int s_corr[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float lsum = 0.f;
  int csum = 0;
  for (int b = warp; b < B; b += nw) {
    const float* row = logits + (size_t)b * K;
    const long long y = labels[b];
    const float l = warp_ce_ls(row, K, y, eps, grad_scale / (float)B, dlogits ? dlogits + (size_t)b * K : nullptr, round);
    // top-1: the first maximum of the row
    float best = -INFINITY;
    int am = 0;
    for (int k = lane; k < K; k += 32) {
      const float v = row[k];
      if (v > best) { best = v; am = k; }
    }
    warp_argmax(best, am);
    if (lane == 0) {
      lsum += l;
      csum += (am == y);
    }
  }
  const float t = block_sum(lsum, s_loss);     // lsum, csum are 0 outside lane 0
  const int c = block_sum(csum, s_corr);
  if (threadIdx.x == 0) {
    loss[0] = t / (float)B;
    if (correct) correct[0] = c;
  }
}

__global__ void sgd_momentum_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf,
                                    size_t n, float lr, float momentum, float wd, float grad_scale, int first) {
  const size_t n4 = n / 4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 pv = reinterpret_cast<float4*>(p)[i];
    const float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 bv = first ? make_float4(0.f, 0.f, 0.f, 0.f) : reinterpret_cast<float4*>(buf)[i];
    float gx = fmaf(wd, pv.x, gv.x * grad_scale), gy = fmaf(wd, pv.y, gv.y * grad_scale);
    float gz = fmaf(wd, pv.z, gv.z * grad_scale), gw = fmaf(wd, pv.w, gv.w * grad_scale);
    bv.x = first ? gx : fmaf(momentum, bv.x, gx);
    bv.y = first ? gy : fmaf(momentum, bv.y, gy);
    bv.z = first ? gz : fmaf(momentum, bv.z, gz);
    bv.w = first ? gw : fmaf(momentum, bv.w, gw);
    pv.x -= lr * bv.x; pv.y -= lr * bv.y; pv.z -= lr * bv.z; pv.w -= lr * bv.w;
    reinterpret_cast<float4*>(buf)[i] = bv;
    reinterpret_cast<float4*>(p)[i] = pv;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (size_t i = n4 * 4; i < n; ++i) {
      const float gg = fmaf(wd, p[i], g[i] * grad_scale);
      const float b = first ? gg : fmaf(momentum, buf[i], gg);
      buf[i] = b;
      p[i] -= lr * b;
    }
  }
}

// torch.optim.Adam (L2 weight decay folded into the gradient, bias-corrected moments)
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, size_t n, float lr, float b1, float b2, float eps, float wd,
                            float grad_scale, float bc1, float bc2) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float pv = p[i];
    const float gg = fmaf(wd, pv, g[i] * grad_scale);
    const float mm = b1 * m[i] + (1.f - b1) * gg;
    const float vv = b2 * v[i] + (1.f - b2) * gg * gg;
    m[i] = mm;
    v[i] = vv;
    const float denom = sqrtf(vv) / sqrtf(bc2) + eps;
    p[i] = pv - (lr / bc1) * mm / denom;
  }
}

// ToTensor + Normalize (dataset/transforms.py:14-19, test.py:80-85) on the GPU: uint8 HWC -> fp32 NCHW, (x/255 - mean)/std
__global__ void normalize_u8_kernel(const unsigned char* __restrict__ x, float* __restrict__ y, size_t npix, size_t hw,
                                    float m0, float m1, float m2, float i0, float i1, float i2) {
  for (size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x; p < npix; p += (size_t)gridDim.x * blockDim.x) {
    const size_t n = p / hw, q = p - n * hw;
    const unsigned char* s = x + p * 3;
    float* d = y + n * 3 * hw + q;
    d[0] = normalize_u8_value(s[0], m0, i0);
    d[hw] = normalize_u8_value(s[1], m1, i1);
    d[2 * hw] = normalize_u8_value(s[2], m2, i2);
  }
}

}  // namespace hk

using namespace hk;

extern "C" {

/* y[B,N] = x[B,F] . w[N,F]^T + bias   via split-K wgmma GEMM; workspace = S*B*N floats */
static int linear_splits(int F) {
  int S = F / 1024;
  if (S < 1) S = 1;
  if (S > 512) S = 512;
  while (F % S != 0 || (F / S) % 4 != 0) {
    if (--S <= 1) return 1;
  }
  return S;
}

size_t hk_linear_fwd_workspace_bytes(int B, int F, int N) { return (size_t)linear_splits(F) * B * N * sizeof(float); }

int hk_linear_fwd(const float* x, const float* w, const float* bias, float* y, int B, int F, int N, void* workspace,
                  size_t workspace_bytes, void* stream) {
  HK_REQUIRE(x && w && y, HK_ERR_ARG, "hk_linear_fwd: null pointer");
  HK_REQUIRE(F % 4 == 0, HK_ERR_UNSUPPORTED, "hk_linear_fwd: in_features=%d must be a multiple of 4", F);
  const int S = linear_splits(F);
  HK_REQUIRE(workspace && workspace_bytes >= (size_t)S * B * N * sizeof(float), HK_ERR_WORKSPACE,
             "hk_linear_fwd: workspace too small");
  return gemm_splitk(x, 0, F, w, 0, F, B, N, F, S, static_cast<float*>(workspace), y, N, N, bias, false,
                     (cudaStream_t)stream);
}

/* dx[B,F] = dy[B,N] . w[N,F] */
int hk_linear_dgrad(const float* dy, const float* w, float* dx, int B, int F, int N, void* stream) {
  HK_REQUIRE(dy && w && dx, HK_ERR_ARG, "hk_linear_dgrad: null pointer");
  HK_REQUIRE(N % 4 == 0 && F % 4 == 0, HK_ERR_UNSUPPORTED, "hk_linear_dgrad: N=%d, F=%d must be multiples of 4", N, F);
  GemmEpi e = {};
  e.C = dx; e.ldc = F; e.alpha = 1.f;
  return gemm_tf32(dy, 0, N, 0, w, 1, F, 0, e, B, F, N, 1, (cudaStream_t)stream);
}

/* dw[N,F] = dy[B,N]^T . x[B,F] ; db[N] = sum_b dy[b,:] */
int hk_linear_wgrad(const float* dy, const float* x, float* dw, float* db, int B, int F, int N, void* stream) {
  HK_REQUIRE(dy && x && dw, HK_ERR_ARG, "hk_linear_wgrad: null pointer");
  HK_REQUIRE(N % 4 == 0 && F % 4 == 0, HK_ERR_UNSUPPORTED, "hk_linear_wgrad: N=%d, F=%d must be multiples of 4", N, F);
  GemmEpi e = {};
  e.C = dw; e.ldc = F; e.alpha = 1.f;
  int r = gemm_tf32(dy, 1, N, 0, x, 1, F, 0, e, N, F, B, 1, (cudaStream_t)stream);
  if (r || !db) return r;
  // db = column sums of dy [B,N]: the B rows are B "partials" of one row of N
  return sum_splits(dy, B, N, 1, N, N, db, N, nullptr, false, (cudaStream_t)stream);
}

int hk_softmax_ce_ls(const float* logits, const long long* labels, float* loss, float* dlogits, int* correct, int B,
                     int K, float label_smoothing, float grad_scale, void* stream) {
  HK_REQUIRE(logits && labels && loss, HK_ERR_ARG, "hk_softmax_ce_ls: null pointer");
  softmax_ce_ls_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(logits, labels, loss, dlogits, correct, B, K,
                                                           label_smoothing, grad_scale, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("softmax_ce_ls_kernel");
  return 0;
}

int hk_normalize_u8(const unsigned char* x_nhwc, float* y_nchw, int N, int H, int W, float mean0, float mean1, float mean2,
                    float std0, float std1, float std2, void* stream) {
  HK_REQUIRE(x_nhwc && y_nchw && N > 0 && H > 0 && W > 0, HK_ERR_ARG, "hk_normalize_u8: bad args");
  HK_REQUIRE(std0 > 0.f && std1 > 0.f && std2 > 0.f, HK_ERR_ARG, "hk_normalize_u8: std must be positive");
  const size_t hw = (size_t)H * W, npix = hw * N;
  normalize_u8_kernel<<<grid_1d(npix, 256), 256, 0, (cudaStream_t)stream>>>(x_nhwc, y_nchw, npix, hw, mean0, mean1, mean2,
                                                                            1.f / std0, 1.f / std1, 1.f / std2);
  HK_LAUNCH_CHECK("normalize_u8_kernel");
  return 0;
}

int hk_sgd_momentum(float* p, const float* g, float* buf, size_t n, float lr, float momentum, float weight_decay,
                    float grad_scale, int first_step, void* stream) {
  HK_REQUIRE(p && g && buf, HK_ERR_ARG, "hk_sgd_momentum: null pointer");
  HK_REQUIRE(aligned16(p) && aligned16(g) && aligned16(buf), HK_ERR_ALIGN, "hk_sgd_momentum: unaligned pointer");
  sgd_momentum_kernel<<<grid_1d(n / 4 + 1, 256), 256, 0, (cudaStream_t)stream>>>(p, g, buf, n, lr, momentum,
                                                                                 weight_decay, grad_scale, first_step);
  HK_LAUNCH_CHECK("sgd_momentum_kernel");
  return 0;
}

int hk_adam(float* p, const float* g, float* m, float* v, size_t n, float lr, float beta1, float beta2, float eps,
            float weight_decay, float grad_scale, int step, void* stream) {
  HK_REQUIRE(p && g && m && v && step >= 1, HK_ERR_ARG, "hk_adam: bad args");
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  adam_kernel<<<grid_1d(n, 256), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay,
                                                                 grad_scale, bc1, bc2);
  HK_LAUNCH_CHECK("adam_kernel");
  return 0;
}

}  // extern "C"
