// Fused bilinear (second-order) pooling kernels.
//
// Reference semantics (model/methods/BCNN.py:13-27):
//     G = X X^T / HW ; z = sqrt(G + 1e-5) ; y = z / max(||z||_2, 1e-12)          X: [B, C, HW]
// and for compact bilinear pooling (model/methods/CBCNN.py:96-135) the Tensor-Sketch of the
// un-normalised Gram, which equals the signed scatter  out[(h1[i]+h2[j]) mod d] += s1[i] s2[j] (X X^T)[i][j].
//
// Design: the C x C Gram X X^T runs on the generic wgmma TF32 GEMM (gemm.cu; HW is the K dimension, X is read straight
// from the NCHW feature map) and small kernels finish it:
//   * hk_bilinear_pool_fwd : closed-form norm from the channel sums, then the Gram with sqrt + L2 normalise in its epilogue;
//   * hk_bilinear_pool_bwd : Gram whose epilogue writes S = (dY+dY^T)/(2z) (z recomputed) and <dY, z>, then the S.X
//                            contraction on the same GEMM, with the rank-1 correction in its epilogue;
//   * hk_cbp_fwd           : Gram whose epilogue scatters into the d sketch bins.
// The C x C Gram itself is never stored.
#include <stdlib.h>

#include "common.cuh"
#include "host.h"
#include "gemm.h"
#include "../../include/hawkeye_b200.h"

namespace hk {



// ---------------------------------------------------------------- K0: per-location channel-sum partials
// partial[b][cs][p] = sum_{c in split cs} x[b][c][p];  also zeroes the per-image scalars used by the backward.
__global__ void colsum_partial_kernel(const float* __restrict__ X, float* __restrict__ partial, int C, int HW, int CS,
                                      float* zero_a, float* zero_b, int zero_n, unsigned keep_mask = 0xffffe000u) {
  extern __shared__ float red[];  // [nrl][HW]
  const int b = blockIdx.x, cs = blockIdx.y;
  if (cs == 0 && threadIdx.x < zero_n) {
    if (zero_a) zero_a[b * zero_n + threadIdx.x] = 0.f;
    if (zero_b) zero_b[b * zero_n + threadIdx.x] = 0.f;
  }
  const int cper = (C + CS - 1) / CS;
  const int c0 = cs * cper, c1 = min(C, c0 + cper);
  const int Q = HW / 4;                                   // float4 columns per row (HW % 4 == 0)
  const int nrl = (int)blockDim.x / Q > 0 ? (int)blockDim.x / Q : 1;  // row lanes
  const int rl = nrl > 1 ? (int)threadIdx.x / Q : 0;
  const float4* xb = reinterpret_cast<const float4*>(X + (size_t)b * C * HW);
  if (rl < nrl) {
    for (int q = nrl > 1 ? (int)threadIdx.x % Q : (int)threadIdx.x; q < Q; q += (nrl > 1 ? Q : (int)blockDim.x)) {
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
      for (int c = c0 + rl; c < c1; c += nrl) {
        // sum what the tensor core will see: kind::tf32 truncates the low 13 mantissa bits
        const float4 v = __ldg(xb + (size_t)c * Q + q);
        s.x += __uint_as_float(__float_as_uint(v.x) & keep_mask);
        s.y += __uint_as_float(__float_as_uint(v.y) & keep_mask);
        s.z += __uint_as_float(__float_as_uint(v.z) & keep_mask);
        s.w += __uint_as_float(__float_as_uint(v.w) & keep_mask);
      }
      reinterpret_cast<float4*>(red + (size_t)rl * HW)[q] = s;
    }
  }
  __syncthreads();
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    float s = 0.f;
    for (int r = 0; r < nrl; ++r) s += red[(size_t)r * HW + p];
    partial[((size_t)b * CS + cs) * HW + p] = s;
  }
}

static inline int pad4(int v) { return (v + 3) & ~3; }

constexpr int COLSUM_SPLITS = 16;
constexpr int COLSUM_SMEM_MAX = 227 * 1024;   // largest dynamic shared memory a block may opt in to on sm_90
// bytes of colsum_partial_kernel's row-lane buffer for a (padded) H*W: HW floats once H*W >= 1024, so H*W <= 58112
static inline size_t colsum_smem(int HW) {
  const int Q = HW / 4;
  const int nrl = 256 / Q > 0 ? 256 / Q : 1;
  return (size_t)nrl * HW * sizeof(float);
}

// bins[b][(h1[i]+h2[j]) mod d] += s1[i] s2[j] G[b][i][j]
static int check_gram_shape(const char* op, const float* X, int B, int C, int HW) {
  HK_REQUIRE(X, HK_ERR_ARG, "%s: null input", op);
  HK_REQUIRE(B > 0 && B <= 65535 && C > 0 && HW > 0, HK_ERR_ARG, "%s: bad shape B=%d C=%d HW=%d", op, B, C, HW);
  HK_REQUIRE(C % 128 == 0, HK_ERR_UNSUPPORTED, "%s: C=%d must be a multiple of 128", op, C);
  HK_REQUIRE(aligned16(X), HK_ERR_ALIGN, "%s: input not 16-byte aligned", op);
  return 0;
}

// the bilinear entry points also reduce each image's channel sums in shared memory
static int check_bilinear_shape(const char* op, const float* X, int B, int C, int HW) {
  if (int r = check_gram_shape(op, X, B, C, HW)) return r;
  HK_REQUIRE(colsum_smem(pad4(HW)) <= (size_t)COLSUM_SMEM_MAX, HK_ERR_UNSUPPORTED,
             "%s: H*W=%d above 58112: the channel sums do not fit in shared memory", op, HW);
  return 0;
}

// [rows][HW] -> [rows][HWp] zero-padded (TMA needs a 16-byte row pitch: H*W = 49 of a 224x224 input becomes 52); zero
// columns change neither the Gram nor the channel sums, and every normalisation keeps using the true H*W
__global__ void pad_cols_kernel(const float* __restrict__ x, float* __restrict__ xp, size_t rows, int HW, int HWp) {
  const size_t total = rows * HWp;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / HWp;
    const int c = (int)(i - r * HWp);
    xp[i] = c < HW ? x[r * HW + c] : 0.f;
  }
}
__global__ void unpad_cols_kernel(const float* __restrict__ xp, float* __restrict__ x, size_t rows, int HW, int HWp) {
  const size_t total = rows * HW;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / HW;
    const int c = (int)(i - r * HW);
    x[i] = xp[r * HWp + c];
  }
}
static int launch_pad(const float* x, float* xp, size_t rows, int HW, cudaStream_t st) {
  pad_cols_kernel<<<H100_SMS * 8, 256, 0, st>>>(x, xp, rows, HW, pad4(HW));
  HK_LAUNCH_CHECK("pad_cols_kernel");
  return 0;
}
static int launch_unpad(const float* xp, float* x, size_t rows, int HW, cudaStream_t st) {
  unpad_cols_kernel<<<H100_SMS * 8, 256, 0, st>>>(xp, x, rows, HW, pad4(HW));
  HK_LAUNCH_CHECK("unpad_cols_kernel");
  return 0;
}

// per-batch scalars for the bilinear backward epilogue:  alpha = 1/(n HW),  beta = -(c_raw/n^2) / (n HW)
__global__ void bilinear_bwd_scalars_kernel(const float* inv_norm, const double* c_raw, float inv_hw, float* alpha,
                                            float* beta, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) {
    const float in = inv_norm[b];
    alpha[b] = in * inv_hw;
    beta[b] = -((float)c_raw[b] * in * in) * in * inv_hw;
  }
}

// s[b][p] = sum over splits of partial
__global__ void colsum_finish_kernel(const float* partial, float* s, int CS, int HW) {
  const int b = blockIdx.x;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    float t = 0.f;
    for (int cs = 0; cs < CS; ++cs) t += partial[((size_t)b * CS + cs) * HW + p];
    s[(size_t)b * HW + p] = t;
  }
}

__global__ void norm_from_s_kernel(const float* s, float* inv_norm, int C, int HW, float inv_hw) {
  const int b = blockIdx.x;
  __shared__ float red[32];
  float acc = 0.f;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const float v = s[(size_t)b * HW + p];
    acc = fmaf(v, v, acc);
  }
  const float t = block_sum(acc, red);
  if (threadIdx.x == 0) {
    const float nrm = sqrtf(t * inv_hw + (float)C * (float)C * 1e-5f);
    inv_norm[b] = 1.f / fmaxf(nrm, 1e-12f);
  }
}

}  // namespace hk

namespace hk {
static int bilinear_bwd_impl(const float* x, const float* dy, float* dx, int B, int C, int HW, float inv_hw, float* S,
                             float* partial, float* svec, float* invn, double* craw, float* alpha, float* beta,
                             cudaStream_t stream);
}

using namespace hk;

extern "C" {

size_t hk_bilinear_pool_fwd_workspace_bytes(int B, int C, int HW) {
  // channel-sum partials [B][CS][HWp] + channel sums [B][HWp] + inv_norm [B] (+ the zero-padded copy of x when H*W % 4 != 0)
  const int HWp = pad4(HW);
  return ((size_t)B * COLSUM_SPLITS * HWp + (size_t)B * HWp + pad4(B) + (HWp != HW ? (size_t)B * C * HWp : 0)) *
         sizeof(float);
}

int hk_bilinear_pool_fwd(const float* x, float* y, float* inv_norm_out, int B, int C, int HW, void* workspace,
                         size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_bilinear_shape("hk_bilinear_pool_fwd", x, B, C, HW);
  if (r) return r;
  HK_REQUIRE(y && aligned16(y), HK_ERR_ALIGN, "hk_bilinear_pool_fwd: output null/unaligned");
  HK_REQUIRE(workspace && workspace_bytes >= hk_bilinear_pool_fwd_workspace_bytes(B, C, HW), HK_ERR_WORKSPACE,
             "hk_bilinear_pool_fwd: workspace too small");
  if ((r = allow_dynamic_smem<colsum_partial_kernel>(COLSUM_SMEM_MAX, "colsum_partial_kernel"))) return r;
  const float inv_hw = 1.f / (float)HW;              // normalisations use the true H*W ...
  const int HWp = pad4(HW);
  float* partial = static_cast<float*>(workspace);
  float* svec = partial + (size_t)B * COLSUM_SPLITS * HWp;
  float* invn_ws = svec + (size_t)B * HWp;
  float* invn = inv_norm_out ? inv_norm_out : invn_ws;
  if (HWp != HW) {                                   // ... the kernels' geometry the padded one
    float* xp = invn_ws + pad4(B);                    // 16-byte aligned: TMA reads it
    if ((r = launch_pad(x, xp, (size_t)B * C, HW, stream))) return r;
    x = xp;
    HW = HWp;
  }
  // The norm in closed form, before the Gram exists: ||z||^2 = sum_ij (G_ij / HW + eps) = sum_p (sum_c x_cp)^2 / HW +
  // C^2 eps, from the channel sums of what the tensor core sees (tf32 mode: truncated operands).  The Gram GEMM's epilogue
  // then writes y = sqrt(G / HW + eps) / ||z|| directly: the C x C Gram never makes a round trip through memory.
  colsum_partial_kernel<<<dim3(B, COLSUM_SPLITS), 256, colsum_smem(HW), stream>>>(x, partial, C, HW, COLSUM_SPLITS, nullptr,
                                                                                nullptr, 0, precise() ? 0xffffffffu : 0xffffe000u);
  HK_LAUNCH_CHECK("colsum_partial_kernel");
  colsum_finish_kernel<<<B, 256, 0, stream>>>(partial, svec, COLSUM_SPLITS, HW);
  HK_LAUNCH_CHECK("colsum_finish_kernel");
  norm_from_s_kernel<<<B, 256, 0, stream>>>(svec, invn, C, HW, inv_hw);
  HK_LAUNCH_CHECK("norm_from_s_kernel");
  GemmEpi e = {};
  e.C = y; e.ldc = C; e.strideC = (long long)C * C;
  e.alpha = inv_hw; e.post_scale = invn; e.post_eps = 1e-5f;
  e.relu = precise() ? 0 : 2;                        // tf32 mode: rounded, y is the operand of the classifier GEMM
  return gemm_tf32(x, 0, HW, (long long)C * HW, x, 0, HW, (long long)C * HW, e, C, C, HW, B, stream);
}

size_t hk_bilinear_pool_bwd_workspace_bytes(int B, int C, int HW) {
  // S [B,C,C] + partial [B,CS,HWp] + s [B,HWp] + inv_norm, c_raw (fp64), alpha, beta [5B] (+ padded copies of x and dx when H*W % 4 != 0)
  const int HWp = pad4(HW);
  return ((size_t)B * C * C + (size_t)B * COLSUM_SPLITS * HWp + (size_t)B * HWp + 5 * (size_t)pad4(B) + 64 +
          (HWp != HW ? 2 * (size_t)B * C * HWp : 0)) * sizeof(float);
}

int hk_bilinear_pool_bwd(const float* x, const float* dy, float* dx, int B, int C, int HW, void* workspace,
                         size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_bilinear_shape("hk_bilinear_pool_bwd", x, B, C, HW);
  if (r) return r;
  HK_REQUIRE(dy && dx && aligned16(dy) && aligned16(dx), HK_ERR_ALIGN, "hk_bilinear_pool_bwd: null/unaligned pointer");
  HK_REQUIRE(workspace && workspace_bytes >= hk_bilinear_pool_bwd_workspace_bytes(B, C, HW), HK_ERR_WORKSPACE,
             "hk_bilinear_pool_bwd: workspace too small");
  if ((r = allow_dynamic_smem<colsum_partial_kernel>(COLSUM_SMEM_MAX, "colsum_partial_kernel"))) return r;
  const float inv_hw = 1.f / (float)HW;
  const int HW_true = HW, HWp = pad4(HW);
  float* S = static_cast<float*>(workspace);
  float* partial = S + (size_t)B * C * C;
  float* svec = partial + (size_t)B * COLSUM_SPLITS * HWp;
  float* invn = svec + (size_t)B * HWp;
  double* craw = reinterpret_cast<double*>(invn + pad4(B));      // 16-byte aligned: every block before it is a multiple of 4 floats
  float* alpha = invn + 3 * pad4(B);
  float* beta = alpha + pad4(B);
  float* dx_out = dx;
  if (HWp != HW) {      // zero-padded copy of x; dx is produced padded and copied back at the end
    float* xp = beta + pad4(B) + 64;
    dx = xp + (size_t)B * C * HWp;
    if ((r = launch_pad(x, xp, (size_t)B * C, HW, stream))) return r;
    x = xp;
    HW = HWp;
  }
  r = bilinear_bwd_impl(x, dy, dx, B, C, HW, inv_hw, S, partial, svec, invn, craw, alpha, beta, stream);
  if (r || dx == dx_out) return r;
  return launch_unpad(dx, dx_out, (size_t)B * C, HW_true, stream);
}

}  // extern "C"

namespace hk {
static int bilinear_bwd_impl(const float* x, const float* dy, float* dx, int B, int C, int HW, float inv_hw, float* S,
                             float* partial, float* svec, float* invn, double* craw, float* alpha, float* beta,
                             cudaStream_t stream) {
  int r;
  // tf32 mode: the column sums see what the tensor core sees (truncated operands); the launch also zeroes c_raw
  colsum_partial_kernel<<<dim3(B, COLSUM_SPLITS), 256, colsum_smem(HW), stream>>>(x, partial, C, HW, COLSUM_SPLITS,
                                                                                reinterpret_cast<float*>(craw), nullptr, 2,
                                                                                precise() ? 0xffffffffu : 0xffffe000u);
  HK_LAUNCH_CHECK("colsum_partial_kernel");
  colsum_finish_kernel<<<B, 256, 0, stream>>>(partial, svec, COLSUM_SPLITS, HW);
  HK_LAUNCH_CHECK("colsum_finish_kernel");
  norm_from_s_kernel<<<B, 256, 0, stream>>>(svec, invn, C, HW, inv_hw);      // closed-form 1/||z||, as in the forward
  HK_LAUNCH_CHECK("norm_from_s_kernel");
  // S = (dY + dY^T) / (2 z) and c_raw = <dY, z> straight from the Gram accumulators (z recomputed in the epilogue)
  GemmEpi e = {};
  e.C = S; e.ldc = C; e.strideC = (long long)C * C;
  e.alpha = inv_hw; e.post_eps = 1e-5f;
  e.mode = EPI_BILINEAR_S; e.dY = dy; e.c_raw = craw;
  if ((r = gemm_tf32(x, 0, HW, (long long)C * HW, x, 0, HW, (long long)C * HW, e, C, C, HW, B, stream))) return r;
  bilinear_bwd_scalars_kernel<<<(B + 127) / 128, 128, 0, stream>>>(invn, craw, inv_hw, alpha, beta, B);
  HK_LAUNCH_CHECK("bilinear_bwd_scalars_kernel");
  // dX = alpha_b * (S . X) + beta_b * 1 s^T      (M=C, K=C, N=HW; X is the MN-major B operand); in tf32 mode rounded: it is
  // the dY operand of the last conv's dgrad / wgrad MMAs
  e = {};
  e.C = dx; e.ldc = HW; e.strideC = (long long)C * HW;
  e.alpha = 1.f; e.alpha_vec = alpha;
  e.D = svec; e.ldd = 0; e.strideD = HW;             // ldd 0: the row s^T is added to every row
  e.beta = 1.f; e.beta_vec = beta;
  e.relu = precise() ? 0 : 2;
  return gemm_tf32(S, 0, C, (long long)C * C, x, 1, HW, (long long)C * HW, e, C, HW, C, B, stream);
}
}  // namespace hk


// =====================================================================================================
// Compact bilinear pooling (reference model/methods/CBCNN.py:96-135) via the Gram-scatter identity:
//   sum_p ifft(fft(x_p S1) * fft(x_p S2)).real [k]  ==  sum_{i,j : (h1[i]+h2[j]) mod d = k} s1[i] s2[j] (X X^T)[i][j]
// so the forward is the same Gram, scattered into the d bins by its epilogue (never stored), followed by
// signed-sqrt (eps 1e-10, CBCNN.py:132) + L2 normalise (:133); no [B*HW, d] sketch or FFT intermediates are formed.
// =====================================================================================================
namespace hk {

// y = normalize(sign(pre) * sqrt(|pre| + 1e-10)); one block per image
__global__ void cbp_finalize_fwd_kernel(const float* __restrict__ pre, float* __restrict__ y, int d, int round) {
  __shared__ float red[32];
  const float* p = pre + (size_t)blockIdx.x * d;
  float acc = 0.f;
  for (int k = threadIdx.x; k < d; k += blockDim.x) acc += fabsf(p[k]) + 1e-10f;   // s_k^2 = |pre_k| + eps (0 if pre==0)
  // sign(0) = 0 in torch: those bins contribute 0, not eps
  float corr = 0.f;
  for (int k = threadIdx.x; k < d; k += blockDim.x) corr += (p[k] == 0.f) ? 1e-10f : 0.f;
  const float n2 = block_sum(acc - corr, red);
  const float inv = 1.f / fmaxf(sqrtf(n2), 1e-12f);
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    const float v = p[k];
    const float s = (v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f)) * sqrtf(fabsf(v) + 1e-10f);
    y[(size_t)blockIdx.x * d + k] = round ? tf32_round(s * inv) : s * inv;
  }
}

// dpre = d/dpre [ normalize(sign(p) sqrt(|p|+eps)) ]^T dy
__global__ void cbp_finalize_bwd_kernel(const float* __restrict__ pre, const float* __restrict__ dy,
                                        float* __restrict__ dpre, int d) {
  __shared__ float red[32];
  const float* p = pre + (size_t)blockIdx.x * d;
  const float* g = dy + (size_t)blockIdx.x * d;
  float n2 = 0.f, dot = 0.f;
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    const float v = p[k];
    if (v != 0.f) {
      const float r = sqrtf(fabsf(v) + 1e-10f);
      n2 += r * r;
      dot += (v > 0.f ? r : -r) * g[k];
    }
  }
  n2 = block_sum(n2, red);
  dot = block_sum(dot, red);
  const float n = fmaxf(sqrtf(n2), 1e-12f);
  const float c = dot / n;                     // <y, dy>
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    const float v = p[k];
    float o = 0.f;
    if (v != 0.f) {
      const float r = sqrtf(fabsf(v) + 1e-10f);
      const float s = v > 0.f ? r : -r;
      const float ds = (g[k] - (s / n) * c) / n;
      o = ds / (2.f * r);
    }
    dpre[(size_t)blockIdx.x * d + k] = o;
  }
}

// S[b][i][j] = dG[i][j] + dG[j][i],  dG[i][j] = s1[i] s2[j] dpre[b][(h1[i]+h2[j]) mod d]
__global__ void cbp_build_s_kernel(const float* __restrict__ dpre, const int* __restrict__ h1,
                                   const int* __restrict__ h2, const float* __restrict__ s1,
                                   const float* __restrict__ s2, float* __restrict__ S, int C, int d, int round) {
  const int b = blockIdx.y;
  const float* dp = dpre + (size_t)b * d;
  const size_t n = (size_t)C * C;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
    const int i = (int)(e / C), j = (int)(e % C);
    int k1 = h1[i] + h2[j];
    if (k1 >= d) k1 -= d;
    int k2 = h1[j] + h2[i];
    if (k2 >= d) k2 -= d;
    const float v = s1[i] * s2[j] * dp[k1] + s1[j] * s2[i] * dp[k2];
    S[(size_t)b * n + e] = round ? tf32_round(v) : v;
  }
}

}  // namespace hk

extern "C" {

int hk_cbp_fwd(const float* x, const int* h1, const int* h2, const float* s1, const float* s2, float* y, float* pre,
               int B, int C, int HW, int d, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_gram_shape("hk_cbp_fwd", x, B, C, HW);
  if (r) return r;
  HK_REQUIRE(h1 && h2 && s1 && s2 && y && pre && d > 0, HK_ERR_ARG, "hk_cbp_fwd: null pointer / bad d");
  Scratch xpad(pad4(HW) != HW ? (size_t)B * C * pad4(HW) * sizeof(float) : 16, stream);   // H*W % 4 != 0 only
  if (pad4(HW) != HW) {
    HK_REQUIRE(xpad.p, HK_ERR_DRIVER, "hk_cbp_fwd: cudaMallocAsync of the padded input failed");
    if ((r = launch_pad(x, xpad.f(), (size_t)B * C, HW, stream))) return r;
    x = xpad.f();
    HW = pad4(HW);
  }
  cudaError_t e = cudaMemsetAsync(pre, 0, (size_t)B * d * sizeof(float), stream);
  if (e != cudaSuccess) return set_error((int)e, "cudaMemsetAsync(pre): %s", cudaGetErrorString(e));
  // the Gram GEMM's epilogue scatters s1[i] s2[j] G_ij into the d bins: the C x C Gram is never stored
  GemmEpi ge = {};
  ge.C = pre; ge.ldc = C; ge.strideC = 0; ge.alpha = 1.f;     // C is not written in EPI_SKETCH mode
  ge.mode = EPI_SKETCH; ge.h1 = h1; ge.h2 = h2; ge.s1 = s1; ge.s2 = s2; ge.bins = pre; ge.d = d;
  if ((r = gemm_tf32(x, 0, HW, (long long)C * HW, x, 0, HW, (long long)C * HW, ge, C, C, HW, B, stream))) return r;
  cbp_finalize_fwd_kernel<<<B, 256, 0, stream>>>(pre, y, d, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("cbp_finalize_fwd_kernel");
  return 0;
}

size_t hk_cbp_bwd_workspace_bytes(int B, int C, int d) { return ((size_t)B * C * C + (size_t)B * d) * sizeof(float); }

int hk_cbp_bwd(const float* x, const float* pre, const float* dy, const int* h1, const int* h2, const float* s1,
               const float* s2, float* dx, int B, int C, int HW, int d, void* workspace, size_t workspace_bytes,
               void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_gram_shape("hk_cbp_bwd", x, B, C, HW);
  if (r) return r;
  HK_REQUIRE(pre && dy && dx && h1 && h2 && s1 && s2 && d > 0, HK_ERR_ARG, "hk_cbp_bwd: null pointer / bad d");
  HK_REQUIRE(workspace && workspace_bytes >= hk_cbp_bwd_workspace_bytes(B, C, d), HK_ERR_WORKSPACE,
             "hk_cbp_bwd: workspace too small");
  const int HWp = pad4(HW);
  Scratch xpad(HWp != HW ? (size_t)B * C * HWp * sizeof(float) : 16, stream);             // H*W % 4 != 0 only
  if (HWp != HW) {
    HK_REQUIRE(xpad.p, HK_ERR_DRIVER, "hk_cbp_bwd: cudaMallocAsync of the padded input failed");
    if ((r = launch_pad(x, xpad.f(), (size_t)B * C, HW, stream))) return r;
    x = xpad.f();
  }
  float* S = static_cast<float*>(workspace);
  float* dpre = S + (size_t)B * C * C;
  cbp_finalize_bwd_kernel<<<B, 256, 0, stream>>>(pre, dy, dpre, d);
  HK_LAUNCH_CHECK("cbp_finalize_bwd_kernel");
  cbp_build_s_kernel<<<dim3(H100_SMS, B), 256, 0, stream>>>(dpre, h1, h2, s1, s2, S, C, d, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("cbp_build_s_kernel");
  // dX = (dG + dG^T) . X      (M = C, K = C, N = HW; X is the MN-major B operand)
  GemmEpi e = {};
  e.C = dx; e.ldc = HW; e.strideC = (long long)C * HW; e.alpha = 1.f;
  e.relu = 2;
  return gemm_tf32(S, 0, C, (long long)C * C, x, 1, HWp, (long long)C * HWp, e, C, HW, C, B, stream);
}

}  // extern "C"
