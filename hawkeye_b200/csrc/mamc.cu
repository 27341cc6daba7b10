// MAMC / N-pairs loss of OSMENet (reference model/loss/MAMC_loss.py:24-90, Sun et al. ECCV 2018, eq. 11).
//
// Reference: features [b, p, D] -> n = b*p anchors, L2-normalised rows, prod = F F^T, and for every anchor i three terms
//     sum_{j in POS} log(1 + sum_{k in NEG} exp(prod[i,k] - prod[i,j]))
// with (POS, NEG) = (same-attention same-class, everything else), (same-attention different-class, different-attention
// different-class), (different-attention same-class, different-attention different-class), built by a Python loop over the
// anchors with repeat()ed [n_pos, n_neg] matrices (MAMC_loss.py:62-88).  Here: sum_k exp(n_k - p_j) = exp(-p_j) * E with
// E = sum_k exp(n_k), so one anchor costs O(n) and the whole loss is ONE launch (one block per anchor) that also emits
// d loss / d prod; the products prod = F F^T and dF = (dprod + dprod^T) F run on the 3xTF32 wgmma GEMM.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

// y = x / max(||x||_2, 1e-12) per row (F.normalize); inv[r] = 1 / max(||x_r||, 1e-12)
__global__ void l2norm_rows_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, float* __restrict__ inv, int D) {
  __shared__ float red[32];
  const float* xr = x + (size_t)blockIdx.x * D;
  float s = 0.f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) s = fmaf(xr[i], xr[i], s);
  s = block_sum(s, red);
  const float iv = 1.f / fmaxf(sqrtf(s), 1e-12f);
  for (int i = threadIdx.x; i < D; i += blockDim.x) y[(size_t)blockIdx.x * D + i] = xr[i] * iv;
  if (threadIdx.x == 0) inv[blockIdx.x] = iv;
}
// dx = inv * (dy - y <y, dy>)
__global__ void l2norm_rows_bwd_kernel(const float* __restrict__ y, const float* __restrict__ inv, const float* __restrict__ dy,
                                       float* __restrict__ dx, int D) {
  __shared__ float red[32];
  const size_t o = (size_t)blockIdx.x * D;
  float s = 0.f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) s = fmaf(y[o + i], dy[o + i], s);
  s = block_sum(s, red);
  const float iv = inv[blockIdx.x];
  for (int i = threadIdx.x; i < D; i += blockDim.x) dx[o + i] = iv * (dy[o + i] - y[o + i] * s);
}

// one block per anchor i.  type of j relative to i: 0 = same attention & same class (includes j = i), 1 = same attention,
// different class, 2 = different attention, same class, 3 = different attention, different class.
//   term A: POS = {0}, NEG = {1,2,3};  term B: POS = {1}, NEG = {3};  term C: POS = {2}, NEG = {3}
// loss_acc (fp64, pre-zeroed) += (A + B + C) / n ;  dprod[i, :] = d(loss)/d(prod[i, :])
__global__ void npair_fwd_bwd_kernel(const float* __restrict__ prod, const int* __restrict__ cls, const int* __restrict__ part,
                                     double* __restrict__ loss_acc, float* __restrict__ dprod, int n) {
  __shared__ float red[32];
  const int i = blockIdx.x;
  const float* pr = prod + (size_t)i * n;
  const int ci = cls[i], pi = part[i];
  float e123 = 0.f, e3 = 0.f;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const int t = (part[j] == pi ? 0 : 2) + (cls[j] == ci ? 0 : 1);
    if (t != 0) {
      const float e = expf(pr[j]);
      e123 += e;
      if (t == 3) e3 += e;
    }
  }
  const float EA = block_sum(e123, red);
  const float EB = block_sum(e3, red);      // NEG of terms B and C is the same set
  // second pass: loss and the POS-side weights  w = E e^{-p} / (1 + E e^{-p}),  W = sum_POS e^{-p} / (1 + E e^{-p})
  float loss = 0.f, WA = 0.f, WB = 0.f, WC = 0.f;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const int t = (part[j] == pi ? 0 : 2) + (cls[j] == ci ? 0 : 1);
    if (t == 3) continue;
    const float em = expf(-pr[j]);
    const float E = t == 0 ? EA : EB;
    const float den = 1.f + E * em;
    loss += log1pf(E * em);
    const float r = em / den;
    if (t == 0) WA += r; else if (t == 1) WB += r; else WC += r;
  }
  loss = block_sum(loss, red);
  WA = block_sum(WA, red);
  WB = block_sum(WB, red);
  WC = block_sum(WC, red);
  const float invn = 1.f / (float)n;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const int t = (part[j] == pi ? 0 : 2) + (cls[j] == ci ? 0 : 1);
    const float p = pr[j];
    const float ep = expf(p), em = expf(-p);
    float g;
    if (t == 0) g = -(EA * em) / (1.f + EA * em);                                   // POS of A
    else if (t == 1) g = ep * WA - (EB * em) / (1.f + EB * em);                     // NEG of A, POS of B
    else if (t == 2) g = ep * WA - (EB * em) / (1.f + EB * em);                     // NEG of A, POS of C
    else g = ep * (WA + WB + WC);                                                   // NEG of A, B and C
    dprod[(size_t)i * n + j] = g * invn;
  }
  if (threadIdx.x == 0) atomicAdd(loss_acc, (double)loss * (double)invn);
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_l2norm_rows_fwd(const float* x, float* y, float* inv_norm, int rows, int D, void* stream) {
  HK_REQUIRE(x && y && inv_norm && rows > 0 && D > 0, HK_ERR_ARG, "hk_l2norm_rows_fwd: bad args");
  l2norm_rows_fwd_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>(x, y, inv_norm, D);
  HK_LAUNCH_CHECK("l2norm_rows_fwd_kernel");
  return 0;
}
int hk_l2norm_rows_bwd(const float* y, const float* inv_norm, const float* dy, float* dx, int rows, int D, void* stream) {
  HK_REQUIRE(y && inv_norm && dy && dx && rows > 0 && D > 0, HK_ERR_ARG, "hk_l2norm_rows_bwd: bad args");
  l2norm_rows_bwd_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>(y, inv_norm, dy, dx, D);
  HK_LAUNCH_CHECK("l2norm_rows_bwd_kernel");
  return 0;
}
int hk_npair_loss(const float* prod, const int* cls, const int* part, double* loss_acc, float* dprod, int n, void* stream) {
  HK_REQUIRE(prod && cls && part && loss_acc && dprod && n > 0, HK_ERR_ARG, "hk_npair_loss: bad args");
  npair_fwd_bwd_kernel<<<n, 128, 0, (cudaStream_t)stream>>>(prod, cls, part, loss_acc, dprod, n);
  HK_LAUNCH_CHECK("npair_fwd_bwd_kernel");
  return 0;
}

}  // extern "C"
