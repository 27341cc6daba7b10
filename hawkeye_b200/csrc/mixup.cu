// Mixup and CutMix of a staged batch (dataset/transforms.py:76-231, dataset/collate_fn.py) and the cross-entropy of the
// soft target they make.  The draws arrive as one row of doubles in device memory (hawkeye_b200/ops_mixup.py documents
// the columns), so a captured step serves every draw and no launch argument changes from batch to batch.  Image i is
// paired with image i - 1 (mod N): the reference's batch.roll(1, 0).
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

enum { MIX_KIND = 0, MIX_LAMBDA = 1, MIX_X1 = 2, MIX_Y1 = 3, MIX_X2 = 4, MIX_Y2 = 5, MIX_WEIGHT = 6, MIX_COLS = 7 };
enum { KIND_MIXUP = 0, KIND_CUTMIX = 1 };

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

template <int V> struct Vec;
template <> struct Vec<1> {
  float v[1];
  __device__ __forceinline__ void load(const float* p) { v[0] = *p; }
  __device__ __forceinline__ void store(float* p) const { *p = v[0]; }
};
template <> struct Vec<4> {
  float v[4];
  __device__ __forceinline__ void load(const float* p) {
    const float4 q = *reinterpret_cast<const float4*>(p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  }
  __device__ __forceinline__ void store(float* p) const {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};

// Each thread owns V consecutive elements at one position of the [C, H, W] image and walks the batch: it keeps image
// n - 1's values in registers while it reads image n, so the batch is read once (image N - 1 twice) and written once.
// Images are read UNROLL at a time, to keep that many loads in flight per thread.
//   Mixup  (transforms.py:133-135): y = fl(fl(x_n (float)lambda) + fl(x_{n-1} (float)(1 - lambda))), the order of
//          batch_rolled.mul_(1 - lambda); batch.mul_(lambda).add_(batch_rolled), with no fused multiply-add.
//   CutMix (transforms.py:225): y = x_{n-1} inside the box, x_n outside.
template <int V>
__global__ void __launch_bounds__(256) mix_batch_kernel(const float* __restrict__ x, const double* __restrict__ mix,
                                                        float* __restrict__ y, int N, size_t chw, int H, int W) {
  constexpr int UNROLL = 4;
  const int kind = (int)mix[MIX_KIND];
  const double lam = mix[MIX_LAMBDA];
  const float a = (float)lam, b = (float)(1.0 - lam);
  // the host checks the box (hk_mix_check); the clamp keeps a bad row from reaching outside the image all the same
  const int x1 = clampi((int)mix[MIX_X1], 0, W), y1 = clampi((int)mix[MIX_Y1], 0, H);
  const int x2 = clampi((int)mix[MIX_X2], 0, W), y2 = clampi((int)mix[MIX_Y2], 0, H);
  const size_t hw = (size_t)H * W;
  for (size_t p = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * V; p < chw; p += (size_t)gridDim.x * blockDim.x * V) {
    bool box[V];
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const size_t r = (p + j) % hw;
      const int h = (int)(r / W), w = (int)(r - (size_t)h * W);
      box[j] = kind == KIND_CUTMIX && h >= y1 && h < y2 && w >= x1 && w < x2;
    }
    Vec<V> prev;
    prev.load(x + (size_t)(N - 1) * chw + p);
    for (int n0 = 0; n0 < N; n0 += UNROLL) {
      Vec<V> cur[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u)
        if (n0 + u < N) cur[u].load(x + (size_t)(n0 + u) * chw + p);
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (n0 + u >= N) break;
        Vec<V> out;
#pragma unroll
        for (int j = 0; j < V; ++j)
          out.v[j] = kind == KIND_MIXUP ? __fadd_rn(__fmul_rn(cur[u].v[j], a), __fmul_rn(prev.v[j], b))
                                        : (box[j] ? prev.v[j] : cur[u].v[j]);
        out.store(y + (size_t)(n0 + u) * chw + p);
        prev = cur[u];
      }
    }
  }
}

// One block; warps stride over rows, as softmax_ce_ls_kernel (head.cu).  Row b's target is w onehot(y_b) +
// (1 - w) onehot(y_{b-1 mod B}) with w = mix[MIX_WEIGHT], each weight rounded to fp32 as the reference's fp32 dense target
// holds it.  A row counts as correct when its first maximum is the target's argmax: the label with the larger weight,
// the lower class index on a tie (target.max(1)[1]).
__global__ void softmax_ce_ls_mix_kernel(const float* __restrict__ logits, const long long* __restrict__ labels,
                                         const double* __restrict__ mix, float* __restrict__ loss,
                                         float* __restrict__ dlogits, int* __restrict__ correct, int B, int K, float eps,
                                         float grad_scale, int round) {
  __shared__ float s_loss[32];
  __shared__ int s_corr[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const double w = mix[MIX_WEIGHT];
  const float wa = (float)w, wb = (float)(1.0 - w);
  float lsum = 0.f;
  int csum = 0;
  for (int b = warp; b < B; b += nw) {
    const float* row = logits + (size_t)b * K;
    const long long ya = labels[b], yb = labels[b == 0 ? B - 1 : b - 1];
    const float l = warp_ce_ls_mix(row, K, ya, wa, yb, wb, eps, grad_scale / (float)B,
                                   dlogits ? dlogits + (size_t)b * K : nullptr, round);
    float best = -INFINITY;
    int am = 0;
    for (int k = lane; k < K; k += 32) {
      const float v = row[k];
      if (v > best) { best = v; am = k; }
    }
    warp_argmax(best, am);
    const long long target = (ya == yb || wa > wb) ? ya : (wb > wa ? yb : (ya < yb ? ya : yb));
    if (lane == 0) {
      lsum += l;
      csum += (am == target);
    }
  }
  const float t = block_sum(lsum, s_loss);     // lsum, csum are 0 outside lane 0
  const int c = block_sum(csum, s_corr);
  if (threadIdx.x == 0) {
    loss[0] = t / (float)B;
    if (correct) correct[0] = c;
  }
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_mix_cols(void) { return MIX_COLS; }

int hk_mix_check(const double* mix, int H, int W) {
  HK_REQUIRE(mix, HK_ERR_ARG, "hk_mix_check: null pointer");
  HK_REQUIRE(H > 0 && W > 0, HK_ERR_ARG, "hk_mix_check: bad H=%d or W=%d", H, W);
  const double kind = mix[MIX_KIND], lam = mix[MIX_LAMBDA], w = mix[MIX_WEIGHT];
  HK_REQUIRE(kind == KIND_MIXUP || kind == KIND_CUTMIX, HK_ERR_ARG, "hk_mix_check: kind %g is neither Mixup (0) nor "
             "CutMix (1)", kind);
  HK_REQUIRE(lam >= 0.0 && lam <= 1.0 && w >= 0.0 && w <= 1.0, HK_ERR_ARG, "hk_mix_check: lambda %g or weight %g "
             "outside [0, 1]", lam, w);
  const double x1 = mix[MIX_X1], y1 = mix[MIX_Y1], x2 = mix[MIX_X2], y2 = mix[MIX_Y2];
  HK_REQUIRE(x1 == (int)x1 && y1 == (int)y1 && x2 == (int)x2 && y2 == (int)y2, HK_ERR_ARG,
             "hk_mix_check: box (%g, %g, %g, %g) is not integral", x1, y1, x2, y2);
  HK_REQUIRE(0 <= x1 && x1 <= x2 && x2 <= W && 0 <= y1 && y1 <= y2 && y2 <= H, HK_ERR_ARG,
             "hk_mix_check: box (%g, %g, %g, %g) lies outside the %d x %d image", x1, y1, x2, y2, W, H);
  return 0;
}

int hk_mix_batch(const float* x, const double* mix, float* y, int N, int C, int H, int W, void* stream) {
  HK_REQUIRE(x && mix && y, HK_ERR_ARG, "hk_mix_batch: null pointer");
  HK_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0, HK_ERR_ARG, "hk_mix_batch: bad N=%d, C=%d, H=%d or W=%d", N, C, H, W);
  HK_REQUIRE(x != y, HK_ERR_ARG, "hk_mix_batch: y must not alias x (image n reads image n - 1)");
  const size_t chw = (size_t)C * H * W;
  if (chw % 4 == 0 && aligned16(x) && aligned16(y)) {
    mix_batch_kernel<4><<<grid_1d(chw / 4, 256), 256, 0, (cudaStream_t)stream>>>(x, mix, y, N, chw, H, W);
  } else {
    mix_batch_kernel<1><<<grid_1d(chw, 256), 256, 0, (cudaStream_t)stream>>>(x, mix, y, N, chw, H, W);
  }
  HK_LAUNCH_CHECK("mix_batch_kernel");
  return 0;
}

int hk_softmax_ce_ls_mix(const float* logits, const long long* labels, const double* mix, float* loss, float* dlogits,
                         int* correct, int B, int K, float label_smoothing, float grad_scale, void* stream) {
  HK_REQUIRE(logits && labels && mix && loss, HK_ERR_ARG, "hk_softmax_ce_ls_mix: null pointer");
  HK_REQUIRE(B > 0 && K > 0, HK_ERR_ARG, "hk_softmax_ce_ls_mix: bad B=%d or K=%d", B, K);
  softmax_ce_ls_mix_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(logits, labels, mix, loss, dlogits, correct, B, K,
                                                               label_smoothing, grad_scale, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("softmax_ce_ls_mix_kernel");
  return 0;
}

}  // extern "C"
