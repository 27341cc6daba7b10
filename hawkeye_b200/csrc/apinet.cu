// Attentive pairwise interaction (reference model/methods/APINet.py, model/loss/APINet_loss.py): pair mining on the device
// (get_pairs + pdist, :76-119), the gather of the mutual-feature pairs and its deterministic adjoint, the attentive gate
// with its four dropouts (:46-61), a stateless counter-based dropout, and the margin-ranking term of the loss (:33-39).
// map1 / map2 / fc run on hk_linear_*, the spatial mean on hk_row_mean_*, the cross-entropy on hk_softmax_ce_ls.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

// splitmix64 output number (call << 40 | i) + 1 of the stream seeded with `seed`; the element is kept when the top 24 bits,
// read as a fraction in [0, 1), are >= p.  Stateless, so the backward re-derives the forward's mask instead of storing it.
// oracle/hop_oracle.py (dropout_keep) restates it in numpy.
__device__ __forceinline__ bool dropout_keep(unsigned long long seed, int call, unsigned long long i, float p) {
  unsigned long long z = seed + ((((unsigned long long)call << 40) | i) + 1ull) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(z >> 40) * 0x1p-24f >= p;
}

__device__ __forceinline__ float drop(float v, bool on, unsigned long long seed, int call, unsigned long long i, float p,
                                      float scale) {
  return !on ? v : (dropout_keep(seed, call, i, p) ? v * scale : 0.f);
}

// One block per row i: <x_i, x_j> and |x_j|^2 by one warp each (lane-strided fmaf, then the fixed xor tree), the distance
// (-2 <x_i, x_j> + |x_j|^2) + |x_i|^2 in the reference's operation order (pdist, APINet.py:116-119), then one thread scans
// j upwards with a strict '<': ties go to the lowest index and a row without candidates keeps index 0 (np.argmin of an
// all-inf row).
__global__ void apinet_pairs_kernel(const float* __restrict__ pool, const long long* __restrict__ labels,
                                    long long* __restrict__ intra, long long* __restrict__ inter,
                                    long long* __restrict__ lab1, long long* __restrict__ lab2, int n, int D) {
  extern __shared__ float sh[];
  float* dot = sh;
  float* nrm = sh + n;
  const int i = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const float* xi = pool + (size_t)i * D;
  for (int j = warp; j < n; j += nw) {
    const float* xj = pool + (size_t)j * D;
    float d = 0.f, q = 0.f;
    for (int k = lane; k < D; k += 32) {
      const float v = xj[k];
      d = fmaf(xi[k], v, d);
      q = fmaf(v, v, q);
    }
    d = warp_sum(d);
    q = warp_sum(q);
    if (lane == 0) { dot[j] = d; nrm[j] = q; }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const float ni = nrm[i];
  const long long li = labels[i];
  int bs = 0, bd = 0;
  float vs = INFINITY, vd = INFINITY;
  for (int j = 0; j < n; ++j) {
    const float dist = __fadd_rn(__fadd_rn(-2.f * dot[j], nrm[j]), ni);
    if (labels[j] == li) {
      if (j != i && dist < vs) { vs = dist; bs = j; }
    } else if (dist < vd) {
      vd = dist;
      bd = j;
    }
  }
  intra[i] = bs;
  inter[i] = bd;
  if (lab1) { lab1[i] = li; lab1[n + i] = li; }
  if (lab2) { lab2[i] = labels[bs]; lab2[n + i] = labels[bd]; }
}

// mutual[r] = [pool[r mod n] | pool[idx2[r]]],  r < 2n  (float4 granularity, D % 4 == 0)
__global__ void apinet_gather_kernel(const float4* __restrict__ pool, const long long* __restrict__ idx2,
                                     float4* __restrict__ mutual, int n, int D4) {
  const size_t total = (size_t)2 * n * 2 * D4;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / (2 * D4));
    const int c = (int)(e - (size_t)r * 2 * D4);
    const long long src = c < D4 ? (r % n) : idx2[r];
    mutual[e] = pool[(size_t)src * D4 + (c < D4 ? c : c - D4)];
  }
}

// dpool[i] = sum of the dmutual halves that were copied from pool[i], taken in ascending row order, the first half of a
// row before its second half: a gather, so no atomics and the same bits on every run.
__global__ void apinet_scatter_kernel(const float4* __restrict__ dmutual, const long long* __restrict__ idx2,
                                      float4* __restrict__ dpool, int n, int D4) {
  extern __shared__ int sidx[];
  for (int r = threadIdx.x; r < 2 * n; r += blockDim.x) sidx[r] = (int)idx2[r];
  __syncthreads();
  const size_t total = (size_t)n * D4;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int i = (int)(e / D4);
    const int c = (int)(e - (size_t)i * D4);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = 0; r < 2 * n; ++r) {
      const size_t row = (size_t)r * 2 * D4;
      if (r % n == i) {
        const float4 v = dmutual[row + c];
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      if (sidx[r] == i) {
        const float4 v = dmutual[row + D4 + c];
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
    dpool[e] = acc;
  }
}

__global__ void dropout_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n, float p, float scale,
                               const long long* __restrict__ seed_ptr, int call) {
  const bool on = p > 0.f;
  const unsigned long long seed = on ? (unsigned long long)seed_ptr[0] : 0ull;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    y[i] = drop(x[i], on, seed, call, i, p, scale);
}

// g1 = sigmoid(m f1), g2 = sigmoid(m f2);  out = [drop(g1 f1 + f1); drop(g2 f2 + f2); drop(g2 f1 + f1); drop(g1 f2 + f2)]
// (self_1, self_2, other_1, other_2: APINet.py:46-69).  Dropout call ids follow the reference's call order:
// call0 + 0: f1_self, +1: f1_other, +2: f2_self, +3: f2_other; the element index is the index within the [2n, D] tensor.
__global__ void apinet_gate_fwd_kernel(const float* __restrict__ m, const float* __restrict__ mutual, float* __restrict__ out,
                                       int rows, int D, float p, float scale, const long long* __restrict__ seed_ptr,
                                       int call0) {
  const bool on = p > 0.f;
  const unsigned long long seed = on ? (unsigned long long)seed_ptr[0] : 0ull;
  const size_t total = (size_t)rows * D;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t r = e / D, d = e - r * D;
    const float f1 = mutual[r * 2 * D + d], f2 = mutual[r * 2 * D + D + d], mv = m[e];
    const float g1 = 1.f / (1.f + expf(-__fmul_rn(mv, f1))), g2 = 1.f / (1.f + expf(-__fmul_rn(mv, f2)));
    out[e] = drop(__fadd_rn(__fmul_rn(g1, f1), f1), on, seed, call0 + 0, e, p, scale);
    out[total + e] = drop(__fadd_rn(__fmul_rn(g2, f2), f2), on, seed, call0 + 2, e, p, scale);
    out[2 * total + e] = drop(__fadd_rn(__fmul_rn(g2, f1), f1), on, seed, call0 + 1, e, p, scale);
    out[3 * total + e] = drop(__fadd_rn(__fmul_rn(g1, f2), f2), on, seed, call0 + 3, e, p, scale);
  }
}

__global__ void apinet_gate_bwd_kernel(const float* __restrict__ m, const float* __restrict__ mutual,
                                       const float* __restrict__ dout, float* __restrict__ dm, float* __restrict__ dmutual,
                                       int rows, int D, float p, float scale, const long long* __restrict__ seed_ptr,
                                       int call0) {
  const bool on = p > 0.f;
  const unsigned long long seed = on ? (unsigned long long)seed_ptr[0] : 0ull;
  const size_t total = (size_t)rows * D;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t r = e / D, d = e - r * D;
    const float f1 = mutual[r * 2 * D + d], f2 = mutual[r * 2 * D + D + d], mv = m[e];
    const float g1 = 1.f / (1.f + expf(-__fmul_rn(mv, f1))), g2 = 1.f / (1.f + expf(-__fmul_rn(mv, f2)));
    const float d1s = drop(dout[e], on, seed, call0 + 0, e, p, scale);
    const float d2s = drop(dout[total + e], on, seed, call0 + 2, e, p, scale);
    const float d1o = drop(dout[2 * total + e], on, seed, call0 + 1, e, p, scale);
    const float d2o = drop(dout[3 * total + e], on, seed, call0 + 3, e, p, scale);
    const float dg1 = d1s * f1 + d2o * f2, dg2 = d1o * f1 + d2s * f2;
    const float da1 = dg1 * g1 * (1.f - g1), da2 = dg2 * g2 * (1.f - g2);
    dm[e] = da1 * f1 + da2 * f2;
    dmutual[r * 2 * D + d] = d1s * (g1 + 1.f) + d1o * (g2 + 1.f) + da1 * mv;
    dmutual[r * 2 * D + D + d] = d2s * (g2 + 1.f) + d2o * (g1 + 1.f) + da2 * mv;
  }
}

// p = softmax(row)[y] as exp(z_y - max) / sum_k exp(z_k - max); also leaves max and the sum for the gradient
__device__ __forceinline__ float warp_softmax_at(const float* __restrict__ row, int K, int y, float& mx, float& se) {
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int k = lane; k < K; k += 32) m = fmaxf(m, row[k]);
  m = warp_max(m);
  float s = 0.f;
  for (int k = lane; k < K; k += 32) s += expf(row[k] - m);
  s = warp_sum(s);
  mx = m;
  se = s;
  return expf(row[y] - m) / s;
}

// MarginRankingLoss(margin)(p_self, p_other, 1) = mean_r max(0, -(p_self - p_other) + margin) over the R pairs (row r, row
// r + R); at the hinge torch's clamp_min passes the gradient (t >= 0).  One block; warp w takes pairs w, w + 32, ...; the
// per-warp fp64 sums are folded in warp order, so the loss is the same on every run.
__global__ void apinet_rank_loss_kernel(const float* __restrict__ logits, const long long* __restrict__ targets,
                                        double* __restrict__ loss_acc, float* __restrict__ dlogits, int R, int K, float margin,
                                        float grad_scale, int round) {
  __shared__ double red[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  double acc = 0.0;
  for (int r = warp; r < R; r += nw) {
    const float* rs = logits + (size_t)r * K;
    const float* ro = logits + (size_t)(r + R) * K;
    const int ys = (int)targets[r], yo = (int)targets[r + R];
    float ms, ss, mo, so;
    const float ps = warp_softmax_at(rs, K, ys, ms, ss);
    const float po = warp_softmax_at(ro, K, yo, mo, so);
    const float t = __fadd_rn(-__fsub_rn(ps, po), margin);
    if (t >= 0.f) {
      acc += (double)t;
      if (dlogits) {
        const float c = grad_scale / (float)R;     // d loss / d p_other = c, d loss / d p_self = -c
        float* gs = dlogits + (size_t)r * K;
        float* go = dlogits + (size_t)(r + R) * K;
        for (int k = lane; k < K; k += 32) {
          const float qs = expf(rs[k] - ms) / ss, qo = expf(ro[k] - mo) / so;
          const float vs = gs[k] - c * ps * ((k == ys ? 1.f : 0.f) - qs);
          const float vo = go[k] + c * po * ((k == yo ? 1.f : 0.f) - qo);
          gs[k] = round ? tf32_round(vs) : vs;
          go[k] = round ? tf32_round(vo) : vo;
        }
      }
    }
  }
  const double s = block_sum(lane == 0 ? acc : 0.0, red);     // every lane of a warp holds its acc
  if (threadIdx.x == 0) loss_acc[0] += s / (double)R;
}

static int check_p(float p, const long long* seed, const char* op) {
  HK_REQUIRE(p >= 0.f && p < 1.f, HK_ERR_ARG, "%s: dropout probability %g outside [0, 1)", op, (double)p);
  HK_REQUIRE(p == 0.f || seed, HK_ERR_ARG, "%s: dropout needs a device seed", op);
  return 0;
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_apinet_pairs(const float* pool, const long long* labels, long long* intra, long long* inter, long long* labels1,
                    long long* labels2, int n, int D, void* stream) {
  HK_REQUIRE(pool && labels && intra && inter, HK_ERR_ARG, "hk_apinet_pairs: null pointer");
  HK_REQUIRE(n >= 2 && n <= 4096 && D > 0, HK_ERR_ARG, "hk_apinet_pairs: n=%d (2..4096), D=%d", n, D);
  apinet_pairs_kernel<<<n, 256, 2 * n * sizeof(float), (cudaStream_t)stream>>>(pool, labels, intra, inter, labels1, labels2,
                                                                                n, D);
  HK_LAUNCH_CHECK("apinet_pairs_kernel");
  return 0;
}

int hk_apinet_gather(const float* pool, const long long* idx2, float* mutual, int n, int D, void* stream) {
  HK_REQUIRE(pool && idx2 && mutual && n > 0 && D > 0, HK_ERR_ARG, "hk_apinet_gather: bad args");
  HK_REQUIRE(D % 4 == 0 && aligned16(pool) && aligned16(mutual), HK_ERR_ALIGN, "hk_apinet_gather: D %% 4, 16-byte rows");
  apinet_gather_kernel<<<grid_1d((size_t)4 * n * D / 4, 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(pool), idx2, reinterpret_cast<float4*>(mutual), n, D / 4);
  HK_LAUNCH_CHECK("apinet_gather_kernel");
  return 0;
}

int hk_apinet_scatter(const float* dmutual, const long long* idx2, float* dpool, int n, int D, void* stream) {
  HK_REQUIRE(dmutual && idx2 && dpool && n > 0 && n <= 4096 && D > 0, HK_ERR_ARG, "hk_apinet_scatter: bad args");
  HK_REQUIRE(D % 4 == 0 && aligned16(dpool) && aligned16(dmutual), HK_ERR_ALIGN, "hk_apinet_scatter: D %% 4, 16-byte rows");
  apinet_scatter_kernel<<<grid_1d((size_t)n * D / 4, 256), 256, 2 * n * sizeof(int), (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(dmutual), idx2, reinterpret_cast<float4*>(dpool), n, D / 4);
  HK_LAUNCH_CHECK("apinet_scatter_kernel");
  return 0;
}

int hk_dropout_fwd(const float* x, float* y, size_t n, float p, const long long* seed, int call, void* stream) {
  HK_REQUIRE(x && y, HK_ERR_ARG, "hk_dropout_fwd: null pointer");
  if (int r = check_p(p, seed, "hk_dropout_fwd")) return r;
  dropout_kernel<<<grid_1d(n, 256), 256, 0, (cudaStream_t)stream>>>(x, y, n, p, 1.f / (1.f - p), seed, call);
  HK_LAUNCH_CHECK("dropout_kernel");
  return 0;
}

int hk_dropout_bwd(const float* dy, float* dx, size_t n, float p, const long long* seed, int call, void* stream) {
  HK_REQUIRE(dy && dx, HK_ERR_ARG, "hk_dropout_bwd: null pointer");
  if (int r = check_p(p, seed, "hk_dropout_bwd")) return r;
  dropout_kernel<<<grid_1d(n, 256), 256, 0, (cudaStream_t)stream>>>(dy, dx, n, p, 1.f / (1.f - p), seed, call);
  HK_LAUNCH_CHECK("dropout_kernel(bwd)");
  return 0;
}

int hk_apinet_gate_fwd(const float* m, const float* mutual, float* out, int rows, int D, float p, const long long* seed,
                       int call0, void* stream) {
  HK_REQUIRE(m && mutual && out && rows > 0 && D > 0, HK_ERR_ARG, "hk_apinet_gate_fwd: bad args");
  if (int r = check_p(p, seed, "hk_apinet_gate_fwd")) return r;
  apinet_gate_fwd_kernel<<<grid_1d((size_t)rows * D, 256), 256, 0, (cudaStream_t)stream>>>(m, mutual, out, rows, D, p,
                                                                                           1.f / (1.f - p), seed, call0);
  HK_LAUNCH_CHECK("apinet_gate_fwd_kernel");
  return 0;
}

int hk_apinet_gate_bwd(const float* m, const float* mutual, const float* dout, float* dm, float* dmutual, int rows, int D,
                       float p, const long long* seed, int call0, void* stream) {
  HK_REQUIRE(m && mutual && dout && dm && dmutual && rows > 0 && D > 0, HK_ERR_ARG, "hk_apinet_gate_bwd: bad args");
  if (int r = check_p(p, seed, "hk_apinet_gate_bwd")) return r;
  apinet_gate_bwd_kernel<<<grid_1d((size_t)rows * D, 256), 256, 0, (cudaStream_t)stream>>>(m, mutual, dout, dm, dmutual, rows,
                                                                                           D, p, 1.f / (1.f - p), seed, call0);
  HK_LAUNCH_CHECK("apinet_gate_bwd_kernel");
  return 0;
}

int hk_apinet_rank_loss(const float* logits, const long long* targets, double* loss_acc, float* dlogits, int R, int K,
                        float margin, float grad_scale, void* stream) {
  HK_REQUIRE(logits && targets && loss_acc && R > 0 && K > 0, HK_ERR_ARG, "hk_apinet_rank_loss: bad args");
  apinet_rank_loss_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(logits, targets, loss_acc, dlogits, R, K, margin, grad_scale,
                                                                precise() ? 0 : 1);
  HK_LAUNCH_CHECK("apinet_rank_loss_kernel");
  return 0;
}

}  // extern "C"
