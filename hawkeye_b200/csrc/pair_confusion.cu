// Pairwise Confusion (reference model/loss/pair_confusion.py, PairwiseConfusionLoss): the label-smoothed cross-entropy of
// every row plus lambda_a times the Euclidean confusion term of the pairs (i, B/2 + i), forward and gradient in one launch.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

// The first maximum of z[0, K) over the warp (the top-1 of hk_softmax_ce_ls).
__device__ __forceinline__ int warp_row_argmax(const float* __restrict__ z, int K) {
  float best = -INFINITY;
  int am = 0;
  for (int k = threadIdx.x & 31; k < K; k += 32) {
    const float v = z[k];
    if (v > best) { best = v; am = k; }
  }
  warp_argmax(best, am);
  return am;
}

// One block; warp w takes the pairs i = w, w + nw, ... (i < B/2) and handles both rows a = i and b = B/2 + i:
//   * the cross-entropy of each row (warp_ce_ls), its gradient (softmax - target) * grad_scale / B written unrounded;
//   * d = z_a - z_b, n = ||d||; when labels differ and n > 0 the term n / B and the gradient +-(lambda / B) d / n
//     (times grad_scale) are added to the two rows, which the same lanes wrote, so no barrier is needed;
//   * the two rows rounded to tf32 once (`round`, the default mode), as hk_softmax_ce_ls stores them.
// pair_confusion.py:23 multiplies the norm by (label_left != label_right); a pair with n = 0 has a zero gradient, as torch's
// norm backward gives it.  The warp partials fold in a fixed order, so the result has the same bits on every run.
__global__ void pc_loss_kernel(const float* __restrict__ logits, const long long* __restrict__ labels,
                               float* __restrict__ loss, float* __restrict__ dlogits, int* __restrict__ correct, int B, int K,
                               float eps, float lambda_a, float grad_scale, int round) {
  __shared__ float s_ce[32], s_pc[32];
  __shared__ int s_corr[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int half = B / 2;
  const float scale = grad_scale / (float)B;
  float ce = 0.f, pc = 0.f;
  int hits = 0;
  for (int i = warp; i < half; i += nw) {
    const size_t ra = (size_t)i * K, rb = (size_t)(half + i) * K;
    const float* za = logits + ra;
    const float* zb = logits + rb;
    float* ga = dlogits + ra;
    float* gb = dlogits + rb;
    const long long ya = labels[i], yb = labels[half + i];
    const float la = warp_ce_ls(za, K, ya, eps, scale, ga, 0);
    const float lb = warp_ce_ls(zb, K, yb, eps, scale, gb, 0);
    const int aa = warp_row_argmax(za, K), ab = warp_row_argmax(zb, K);
    float ss = 0.f;
    for (int k = lane; k < K; k += 32) {
      const float d = za[k] - zb[k];
      ss = fmaf(d, d, ss);
    }
    const float n = sqrtf(warp_sum(ss));
    const bool term = ya != yb && n > 0.f;
    const float c = term ? lambda_a * scale / n : 0.f;
    for (int k = lane; k < K; k += 32) {
      const float d = za[k] - zb[k];
      const float va = fmaf(c, d, ga[k]), vb = fmaf(-c, d, gb[k]);
      ga[k] = round ? tf32_round(va) : va;
      gb[k] = round ? tf32_round(vb) : vb;
    }
    if (lane == 0) {
      ce += la + lb;
      pc += term ? n : 0.f;
      hits += (aa == ya) + (ab == yb);
    }
  }
  const float t_ce = block_sum(ce, s_ce);        // ce, pc, hits are 0 outside lane 0
  const float t_pc = block_sum(pc, s_pc);
  const int c = block_sum(hits, s_corr);
  if (threadIdx.x == 0) {
    loss[0] = fmaf(lambda_a, t_pc / (float)B, t_ce / (float)B);
    correct[0] = c;
  }
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_pc_loss(const float* logits, const long long* labels, float* loss, float* dlogits, int* correct, int B, int K,
               float label_smoothing, float lambda_a, float grad_scale, void* stream) {
  HK_REQUIRE(logits && labels && loss && dlogits && correct, HK_ERR_ARG, "hk_pc_loss: null pointer");
  HK_REQUIRE(B >= 2 && B % 2 == 0 && K > 0, HK_ERR_ARG, "hk_pc_loss: B=%d must be even and at least 2, K=%d > 0", B, K);
  pc_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(logits, labels, loss, dlogits, correct, B, K, label_smoothing,
                                                       lambda_a, grad_scale, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("pc_loss_kernel");
  return 0;
}

}  // extern "C"
