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

// Block exclusive prefix sum in thread order: returns the sum of v over the threads below this one and sets total to
// the sum over all threads.  Same conditions on blockDim.x and red[] as block_sum.
template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* red, T& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  __syncthreads();
  if (lane == 31) red[warp] = inc;
  __syncthreads();
  T below = T(0);
  total = T(0);
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
    if (i < warp) below += red[i];
    total += red[i];
  }
  return below + inc - v;
}

// The softmax statistics of one row segment z[0, K), by one warp: lse = log sum_k exp z[k] and sl = sum_k z[k], in every
// lane.  The one softmax of the cross-entropies below.
__device__ __forceinline__ void warp_lse(const float* __restrict__ z, int K, float& lse, float& sl) {
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int k = lane; k < K; k += 32) m = fmaxf(m, z[k]);
  m = warp_max(m);
  float se = 0.f, s = 0.f;
  for (int k = lane; k < K; k += 32) {
    se += expf(z[k] - m);
    s += z[k];
  }
  se = warp_sum(se);
  sl = warp_sum(s);
  lse = m + logf(se);
}

// Label-smoothed cross-entropy of one row segment z[0, K) with target y (eps = smoothing), by one warp: returns the row's
// loss term and, unless g is null, writes (softmax - target distribution) * scale to g (rounded to tf32 when `round`).  A
// target outside [0, K) gets no one-hot term and z is not read at it.
__device__ __forceinline__ float warp_ce_ls(const float* __restrict__ z, int K, long long y, float eps, float scale,
                                            float* __restrict__ g, int round) {
  const int lane = threadIdx.x & 31;
  float lse, sl;
  warp_lse(z, K, lse, sl);
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

// warp_ce_ls against the soft target wa onehot(ya) + wb onehot(yb) (Mixup / CutMix; ya == yb sums the two weights): the
// loss term (1 - eps) [wa (lse - z[ya]) + wb (lse - z[yb])] + eps (lse - mean(z)), and unless g is null
// (softmax - ((1 - eps) target + eps / K)) * scale written to g.  A label outside [0, K) gets no one-hot term.
__device__ __forceinline__ float warp_ce_ls_mix(const float* __restrict__ z, int K, long long ya, float wa, long long yb,
                                                float wb, float eps, float scale, float* __restrict__ g, int round) {
  const int lane = threadIdx.x & 31;
  float lse, sl;
  warp_lse(z, K, lse, sl);
  const float za = (ya >= 0 && ya < K) ? z[ya] : lse, zb = (yb >= 0 && yb < K) ? z[yb] : lse;
  if (g) {
    for (int k = lane; k < K; k += 32) {
      const float t = ((k == ya ? wa : 0.f) + (k == yb ? wb : 0.f)) * (1.f - eps) + eps / (float)K;
      const float v = (expf(z[k] - lse) - t) * scale;
      g[k] = round ? tf32_round(v) : v;
    }
  }
  return fmaf(1.f - eps, fmaf(wa, lse - za, wb * (lse - zb)), eps * (lse - sl / (float)K));
}

}  // namespace hk
