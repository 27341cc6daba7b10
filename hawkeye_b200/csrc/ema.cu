// Exponential moving average of a model's weights (torch.optim.swa_utils.AveragedModel.update_parameters with
// use_buffers=True and torchvision's ExponentialMovingAverage avg_fn), and the in-place exchange of the model and its
// average for evaluation.  The tensors are segments of a table in device memory (hawkeye_b200/engine.py builds it once):
// one launch covers the flat parameter buffer, the parameters outside it and every buffer.  Each block owns one chunk
// of EMA_CHUNK elements of one segment and finds its segment by a binary search over the segments' first chunks.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

#include <climits>

namespace hk {

enum { EMA_MODEL = 0, EMA_AVG = 1, EMA_N = 2, EMA_KIND = 3, EMA_CHUNK0 = 4, EMA_COLS = 5 };
enum { EMA_F32 = 0, EMA_I64 = 1 };
constexpr int EMA_THREADS = 256;
constexpr int EMA_VECS = 4;                                              // float4 per thread and chunk
constexpr long long EMA_CHUNK = (long long)EMA_THREADS * EMA_VECS * 4;  // elements per block

__device__ __forceinline__ bool dev_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// torch's d * avg + (1 - d) * p on fp32 tensors: two roundings of the products, one of the sum, no contraction.
__device__ __forceinline__ float ema_f32(float e, float p, float d, float omd) {
  return __fadd_rn(__fmul_rn(e, d), __fmul_rn(p, omd));
}

// The same on int64 tensors (num_batches_tracked): a Python float times an int64 tensor promotes to fp32, and copy_
// back into the int64 tensor truncates toward zero.
__device__ __forceinline__ long long ema_i64(long long e, long long p, float d, float omd) {
  return (long long)ema_f32(__ll2float_rn(e), __ll2float_rn(p), d, omd);
}

template <bool SWAP>
__device__ __forceinline__ void ema_f32_elem(float* m, float* e, bool copy, float d, float omd) {
  const float p = *m;
  if (SWAP) {
    *m = *e;
    *e = p;
  } else {
    *e = copy ? p : ema_f32(*e, p, d, omd);
  }
}

__device__ __forceinline__ float4 ema_f32x4(float4 e, float4 p, float d, float omd) {
  return make_float4(ema_f32(e.x, p.x, d, omd), ema_f32(e.y, p.y, d, omd), ema_f32(e.z, p.z, d, omd),
                     ema_f32(e.w, p.w, d, omd));
}

// SWAP = false: e = p when *n_averaged == 0, else e = d e + (1 - d) p.  SWAP = true: exchange m and e.
template <bool SWAP>
__global__ void __launch_bounds__(EMA_THREADS) ema_kernel(const long long* __restrict__ table, int nseg,
                                                          const long long* __restrict__ n_averaged, float d, float omd) {
  const long long b = blockIdx.x;
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (table[(size_t)mid * EMA_COLS + EMA_CHUNK0] <= b) lo = mid; else hi = mid - 1;
  }
  const long long* row = table + (size_t)lo * EMA_COLS;
  const long long base = (b - row[EMA_CHUNK0]) * EMA_CHUNK, n = row[EMA_N];
  const int cnt = (int)min(EMA_CHUNK, n - base);
  const bool copy = !SWAP && *n_averaged == 0;
  if (row[EMA_KIND] == EMA_I64) {
    long long* m = reinterpret_cast<long long*>(row[EMA_MODEL]) + base;
    long long* e = reinterpret_cast<long long*>(row[EMA_AVG]) + base;
    for (int i = threadIdx.x; i < cnt; i += EMA_THREADS) {
      const long long p = m[i];
      if (SWAP) {
        m[i] = e[i];
        e[i] = p;
      } else {
        e[i] = copy ? p : ema_i64(e[i], p, d, omd);
      }
    }
    return;
  }
  float* m = reinterpret_cast<float*>(row[EMA_MODEL]) + base;
  float* e = reinterpret_cast<float*>(row[EMA_AVG]) + base;
  if (!(dev_aligned16(m) && dev_aligned16(e))) {
    for (int i = threadIdx.x; i < cnt; i += EMA_THREADS) ema_f32_elem<SWAP>(m + i, e + i, copy, d, omd);
    return;
  }
  // the flat parameter buffer (and any other 16-byte-aligned segment): every load of the chunk issued before any store
  const int nv = cnt >> 2;
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* e4 = reinterpret_cast<float4*>(e);
  float4 pv[EMA_VECS], ev[EMA_VECS];
#pragma unroll
  for (int k = 0; k < EMA_VECS; ++k) {
    const int i = threadIdx.x + k * EMA_THREADS;
    if (i < nv) pv[k] = m4[i];
    if (i < nv && !copy) ev[k] = e4[i];
  }
  if (copy) {
#pragma unroll
    for (int k = 0; k < EMA_VECS; ++k)
      if (threadIdx.x + k * EMA_THREADS < nv) e4[threadIdx.x + k * EMA_THREADS] = pv[k];
  } else {
#pragma unroll
    for (int k = 0; k < EMA_VECS; ++k) {
      const int i = threadIdx.x + k * EMA_THREADS;
      if (i < nv) {
        if (SWAP) {
          m4[i] = ev[k];
          e4[i] = pv[k];
        } else {
          e4[i] = ema_f32x4(ev[k], pv[k], d, omd);
        }
      }
    }
  }
  const int tail = nv * 4 + threadIdx.x;          // the last chunk of a segment whose length is not a multiple of 4
  if (tail < cnt) ema_f32_elem<SWAP>(m + tail, e + tail, copy, d, omd);
}

// The counter's increment, or torchvision's warm-up reset to 0, in a launch of its own after the update: stream order
// then guarantees that no block of the update reads the new value.
__global__ void ema_count_kernel(long long* n_averaged, int reset) { *n_averaged = reset ? 0 : *n_averaged + 1; }

static int ema_args(const char* what, const long long* table, int nseg, long long nchunks) {
  HK_REQUIRE(table, HK_ERR_ARG, "%s: null pointer", what);
  HK_REQUIRE(nseg > 0 && nchunks > 0 && nchunks <= INT_MAX, HK_ERR_ARG, "%s: bad nseg=%d or nchunks=%lld", what, nseg,
             nchunks);
  return 0;
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_ema_cols(void) { return EMA_COLS; }

long long hk_ema_plan(long long* table, int nseg) {
  HK_REQUIRE(table, HK_ERR_ARG, "hk_ema_plan: null pointer");
  HK_REQUIRE(nseg > 0, HK_ERR_ARG, "hk_ema_plan: bad nseg=%d", nseg);
  long long chunks = 0;
  for (int s = 0; s < nseg; ++s) {
    long long* row = table + (size_t)s * EMA_COLS;
    HK_REQUIRE(row[EMA_MODEL] && row[EMA_AVG], HK_ERR_ARG, "hk_ema_plan: segment %d has a null pointer", s);
    HK_REQUIRE(row[EMA_MODEL] != row[EMA_AVG], HK_ERR_ARG, "hk_ema_plan: segment %d averages into itself", s);
    HK_REQUIRE(row[EMA_N] > 0, HK_ERR_ARG, "hk_ema_plan: segment %d has %lld elements", s, row[EMA_N]);
    HK_REQUIRE(row[EMA_KIND] == EMA_F32 || row[EMA_KIND] == EMA_I64, HK_ERR_ARG,
               "hk_ema_plan: segment %d has kind %lld (0 float32, 1 int64)", s, row[EMA_KIND]);
    const long long esz = row[EMA_KIND] == EMA_I64 ? 8 : 4;
    HK_REQUIRE(row[EMA_MODEL] % esz == 0 && row[EMA_AVG] % esz == 0, HK_ERR_ALIGN,
               "hk_ema_plan: segment %d is not aligned to its %lld-byte elements", s, esz);
    row[EMA_CHUNK0] = chunks;
    chunks += (row[EMA_N] + EMA_CHUNK - 1) / EMA_CHUNK;
    HK_REQUIRE(chunks <= INT_MAX, HK_ERR_ARG, "hk_ema_plan: more than %d chunks of %lld elements", INT_MAX, EMA_CHUNK);
  }
  return chunks;
}

int hk_ema_update(const long long* table, int nseg, long long nchunks, long long* n_averaged, float decay,
                  float one_minus_decay, int reset_after, void* stream) {
  if (int e = ema_args("hk_ema_update", table, nseg, nchunks)) return e;
  HK_REQUIRE(n_averaged, HK_ERR_ARG, "hk_ema_update: null pointer");
  HK_REQUIRE(decay >= 0.f && decay <= 1.f && one_minus_decay >= 0.f && one_minus_decay <= 1.f, HK_ERR_ARG,
             "hk_ema_update: decay %g or 1 - decay %g outside [0, 1]", decay, one_minus_decay);
  ema_kernel<false><<<(unsigned)nchunks, EMA_THREADS, 0, (cudaStream_t)stream>>>(table, nseg, n_averaged, decay,
                                                                                  one_minus_decay);
  HK_LAUNCH_CHECK("ema_kernel");
  ema_count_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(n_averaged, reset_after ? 1 : 0);
  HK_LAUNCH_CHECK("ema_count_kernel");
  return 0;
}

int hk_ema_swap(const long long* table, int nseg, long long nchunks, void* stream) {
  if (int e = ema_args("hk_ema_swap", table, nseg, nchunks)) return e;
  ema_kernel<true><<<(unsigned)nchunks, EMA_THREADS, 0, (cudaStream_t)stream>>>(table, nseg, nullptr, 0.f, 1.f);
  HK_LAUNCH_CHECK("ema_kernel_swap");
  return 0;
}

}  // extern "C"
