// Warp and block reductions of the hawkeye_b200 kernels, and the label-smoothed cross-entropy of one row built on them.
// Part of common.cuh, which includes it after tf32_round: include common.cuh, not this file.
//
// Every reduction folds in a fixed order: the xor tree over the lanes (offsets 16, 8, 4, 2, 1), then, for a block, the
// warp partials in ascending warp order.  So a result has the same bits on every run.
#pragma once

namespace hk {

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Each lane's (best, idx) from its own scan -> in every lane, the warp's maximum and the lowest index that holds it.
__device__ __forceinline__ void warp_argmax(float& best, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oa = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ob > best || (ob == best && oa < idx)) { best = ob; idx = oa; }
  }
}

// Block sum / max over all threads, returned to every thread; red[] holds one partial per warp.  blockDim.x must be a
// multiple of 32 and at most 1024.  The leading barrier lets a block call these back to back on the same red[32].
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  T t = T(0);
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
  return t;
}

__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) t = fmaxf(t, red[i]);
  return t;
}

// Label-smoothed cross-entropy of one row segment z[0, K) with target y (eps = smoothing), by one warp: returns the row's
// loss term and, unless g is null, writes (softmax - target distribution) * scale to g (rounded to tf32 when `round`).  A
// target outside [0, K) gets no one-hot term and z is not read at it.
__device__ __forceinline__ float warp_ce_ls(const float* __restrict__ z, int K, long long y, float eps, float scale,
                                            float* __restrict__ g, int round) {
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int k = lane; k < K; k += 32) m = fmaxf(m, z[k]);
  m = warp_max(m);
  float se = 0.f, sl = 0.f;
  for (int k = lane; k < K; k += 32) {
    se += expf(z[k] - m);
    sl += z[k];
  }
  se = warp_sum(se);
  sl = warp_sum(sl);
  const float lse = m + logf(se);
  const bool valid = y >= 0 && y < K;
  const float zy = valid ? z[y] : lse;
  if (g) {
    for (int k = lane; k < K; k += 32) {
      const float t = (k == y ? (1.f - eps) : 0.f) + eps / (float)K;
      const float v = (expf(z[k] - lse) - t) * scale;
      g[k] = round ? tf32_round(v) : v;
    }
  }
  // (1 - eps) (lse - z[y]) + eps (lse - mean(z)), with the fused multiply-add spelled out: left to the compiler, which
  // product it fuses depends on the kernel this is inlined into
  return fmaf(1.f - eps, lse - zy, eps * (lse - sl / (float)K));
}

}  // namespace hk
