// Fast MPN-COV pooling head (reference model/methods/MPNCOV.py:105-230): covariance pooling, Newton-Schulz matrix
// square root (forward AND the reference's hand-derived backward, formula by formula), upper-triangular vectorise.
//
// Every matrix product runs on the wgmma GEMM (gemm.cu).  The coupled Newton-Schulz chain is 12 dependent 256^3
// products forward / 38 backward and is NOT converged after 5 iterations, so rounding compounds; the
// chain therefore runs in 3xTF32: every matrix is kept as a (hi, lo) pair of tf32 values (hi = rn(x), lo = rn(x-hi))
// and  A.B ~= Ah.Bh + Al.Bh + Ah.Bl  (three tensor-core GEMMs, fp32 accumulation) — fp32-class accuracy at 3x the
// (tiny: 1.8 GFLOP/img) cost.
#include "common.cuh"
#include "host.h"
#include "gemm.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

struct Pair { float* hi; float* lo; };

// C(hi,lo) = alpha * (A.B) + diag*I + beta * D(hi+lo)     A,B,D: [batch][n][n] row-major pairs
static int mm3(Pair A, Pair B, Pair C, int n, int batch, float alpha, float diag, const Pair* D, float beta,
               cudaStream_t st) {
  const long long s = (long long)n * n;
  GemmEpi f = {};
  f.C = C.hi; f.C_lo = C.lo; f.ldc = n; f.strideC = s;
  f.alpha = alpha; f.diag = diag;
  if (D) { f.D = D->hi; f.D_lo = D->lo; f.ldd = n; f.strideD = s; f.beta = beta; }
  // one launch: every k-step issues Ah.Bl, Al.Bh, Ah.Bh into the same accumulators (gemm.cu, triple mode)
  return gemm_tf32_pair(A.hi, A.lo, 0, n, s, B.hi, B.lo, 1, n, s, f, n, n, n, batch, st);
}

// ------------------------------------------------------------------------------------------------ small kernels
// centre the rows of X [B*C][M] (subtract the spatial mean) and round to tf32:  X I_hat X^T = Xc Xc^T / M
__global__ void center_rows_kernel(const float* __restrict__ x, float* __restrict__ xc, int M, int Mp, int round) {
  const size_t row = blockIdx.x;
  const float* p = x + row * M;
  float s = 0.f;
  for (int i = threadIdx.x; i < M; i += 32) s += p[i];
  s = warp_sum(s) / (float)M;
  for (int i = threadIdx.x; i < Mp; i += 32)       // columns M..Mp-1 (pitch padding for TMA) stay zero: they add nothing
    xc[row * Mp + i] = i < M ? (round ? tf32_round(p[i] - s) : p[i] - s) : 0.f;
}

// normA[b] = trace(x[b]); A = x / normA as a (hi, lo) pair
__global__ void trace_normalize_kernel(const float* __restrict__ x, float* __restrict__ normA, float* __restrict__ Ahi,
                                       float* __restrict__ Alo, int n) {
  __shared__ float red[32];
  const float* xb = x + (size_t)blockIdx.x * n * n;
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += xb[(size_t)i * n + i];
  const float tr = block_sum(s, red);
  if (threadIdx.x == 0) normA[blockIdx.x] = tr;
  const float inv = 1.f / tr;
  for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
    const float v = xb[i] * inv;
    const float h = tf32_round(v);
    Ahi[(size_t)blockIdx.x * n * n + i] = h;
    Alo[(size_t)blockIdx.x * n * n + i] = tf32_round(v - h);
  }
}

// out(hi,lo) = alpha * scale_b * (in_hi + in_lo) + diag * I          (in_lo may be null; scale may be null)
__global__ void affine_diag_split_kernel(const float* __restrict__ in_hi, const float* __restrict__ in_lo,
                                         float* __restrict__ out_hi, float* __restrict__ out_lo, float alpha,
                                         const float* __restrict__ scale, int sqrt_scale, float diag, int n, size_t total) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t b = i / ((size_t)n * n);
    const int rc = (int)(i % ((size_t)n * n));
    float sc = scale ? scale[b] : 1.f;
    if (sqrt_scale) sc = sqrtf(sc);
    float v = in_hi[i] + (in_lo ? in_lo[i] : 0.f);
    v = alpha * sc * v + ((rc / n == rc % n) ? diag : 0.f);
    const float h = tf32_round(v);
    out_hi[i] = h;
    out_lo[i] = tf32_round(v - h);
  }
}

// Sqrtm.backward tail (MPNCOV.py:194-201):  D = (tmpD - 0.5 dldZ)^T ; grad = D/normA + (aux - sum(D.x)/normA^2) I
// with aux = sum(g . YZY) / (2 sqrt(normA)) = sum(g . y) / (2 normA)   (y = YZY sqrt(normA) is the saved output)
__global__ void sqrtm_bwd_tail_kernel(const float* __restrict__ tD_hi, const float* __restrict__ tD_lo,
                                      const float* __restrict__ dZ_hi, const float* __restrict__ dZ_lo,
                                      const float* __restrict__ x, const float* __restrict__ y,
                                      const float* __restrict__ g, const float* __restrict__ normA,
                                      float* __restrict__ grad, int n) {
  __shared__ float red[32];
  const size_t off = (size_t)blockIdx.x * n * n;
  float gaux = 0.f, gy = 0.f;
  for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
    const int r = i / n, c = i % n;
    const int t = c * n + r;   // D[r][c] = M[c][r]
    const float d = (tD_hi[off + t] + tD_lo[off + t]) - 0.5f * (dZ_hi[off + t] + dZ_lo[off + t]);
    gaux = fmaf(d, x[off + i], gaux);
    gy = fmaf(g[off + i], y[off + i], gy);
  }
  const float ga = block_sum(gaux, red), gyy = block_sum(gy, red);
  const float na = normA[blockIdx.x];
  const float coef = gyy / (2.f * na) - ga / (na * na);
  for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
    const int r = i / n, c = i % n;
    const int t = c * n + r;
    const float d = (tD_hi[off + t] + tD_lo[off + t]) - 0.5f * (dZ_hi[off + t] + dZ_lo[off + t]);
    grad[off + i] = d / na + (r == c ? coef : 0.f);
  }
}

// out = (hi + lo) * (sqrt_scale ? sqrt(scale[b]) : scale[b])      (scale may be null)
__global__ void pair_combine_scale_kernel(const float* __restrict__ hi, const float* __restrict__ lo,
                                          float* __restrict__ out, const float* __restrict__ scale, int sqrt_scale,
                                          size_t per_batch, size_t total) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float sc = scale ? scale[i / per_batch] : 1.f;
    if (sqrt_scale) sc = sqrtf(sc);
    out[i] = (hi[i] + lo[i]) * sc;
  }
}

// Triuvec (MPNCOV.py:205-230): row-major upper triangle, row r holds columns r..n-1
__global__ void triuvec_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int n) {
  const int r = blockIdx.x, b = blockIdx.y;
  const size_t L = (size_t)n * (n + 1) / 2;
  const size_t base = (size_t)r * n - (size_t)r * (r - 1) / 2;
  for (int c = r + threadIdx.x; c < n; c += blockDim.x) y[b * L + base + (c - r)] = x[((size_t)b * n + r) * n + c];
}
__global__ void triuvec_bwd_kernel(const float* __restrict__ g, float* __restrict__ dx, int n) {
  const int r = blockIdx.x, b = blockIdx.y;
  const size_t L = (size_t)n * (n + 1) / 2;
  const size_t base = (size_t)r * n - (size_t)r * (r - 1) / 2;
  for (int c = threadIdx.x; c < n; c += blockDim.x)
    dx[((size_t)b * n + r) * n + c] = c >= r ? g[b * L + base + (c - r)] : 0.f;
}

}  // namespace hk

using namespace hk;

extern "C" {

/* ---------------- Covpool (MPNCOV.py:105-134) ---------------- */
int hk_covpool_fwd(const float* x, float* cov, float* xc, int B, int C, int M, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  HK_REQUIRE(x && cov && xc, HK_ERR_ARG, "hk_covpool_fwd: null pointer");
  const int Mp = (M + 3) & ~3;                      // xc is [B, C, Mp]: centred rows at a 16-byte pitch
  center_rows_kernel<<<(unsigned)((size_t)B * C), 32, 0, st>>>(x, xc, M, Mp, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("center_rows_kernel");
  GemmEpi e = {};
  e.C = cov; e.ldc = C; e.strideC = (long long)C * C; e.alpha = 1.f / (float)M;
  return gemm_tf32(xc, 0, Mp, (long long)C * Mp, xc, 0, Mp, (long long)C * Mp, e, C, C, Mp, B, st);
}

int hk_covpool_bwd(const float* xc, const float* g, float* dx, int B, int C, int M, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  HK_REQUIRE(xc && g && dx, HK_ERR_ARG, "hk_covpool_bwd: null pointer");
  const int Mp = (M + 3) & ~3;
  // dX = (g + g^T) X I_hat = (g . Xc + g^T . Xc) / M        (xc pitch Mp, dx pitch M)
  GemmEpi e = {};
  e.C = dx; e.ldc = M; e.strideC = (long long)C * M; e.alpha = 1.f;
  int r = gemm_tf32(g, 0, C, (long long)C * C, xc, 1, Mp, (long long)C * Mp, e, C, M, C, B, st);   // raw g . Xc
  if (r) return r;
  e.E = dx;   // (g^T . Xc + g . Xc) / M
  e.alpha = 1.f / (float)M;
  return gemm_tf32(g, 1, C, (long long)C * C, xc, 1, Mp, (long long)C * Mp, e, C, M, C, B, st);
}

/* ---------------- Sqrtm (MPNCOV.py:137-202) ---------------- */
/* saved layout (floats): normA[B padded to 4] | A(hi,lo) | Y_0..Y_{L-1}(hi,lo each) | Z_0..Z_{L-1}(hi,lo each), L = iterN-1 */
size_t hk_sqrtm_saved_floats(int B, int n, int iterN) {
  return (size_t)(2 + 4 * (iterN - 1)) * B * n * n + (((size_t)B + 3) / 4) * 4;
}
size_t hk_sqrtm_fwd_workspace_bytes(int B, int n) { return (size_t)5 * B * n * n * sizeof(float); }
size_t hk_sqrtm_bwd_workspace_bytes(int B, int n) { return (size_t)23 * B * n * n * sizeof(float); }

struct SqrtmSaved {
  float* normA;
  Pair A;
  float* base;
  size_t S;
  int L;
  Pair Y(int i) const { return Pair{base + (2 + 2 * i) * S, base + (3 + 2 * i) * S}; }
  Pair Z(int i) const { return Pair{base + (2 + 2 * L + 2 * i) * S, base + (3 + 2 * L + 2 * i) * S}; }
};
static SqrtmSaved saved_view(float* saved, int B, int n, int iterN) {
  SqrtmSaved v;
  v.S = (size_t)B * n * n;
  v.L = iterN - 1;
  v.normA = saved;
  v.base = saved + (((size_t)B + 3) / 4) * 4;
  v.A = Pair{v.base, v.base + v.S};
  return v;
}

int hk_sqrtm_fwd(const float* x, float* y, float* saved, int B, int n, int iterN, void* workspace,
                 size_t workspace_bytes, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  HK_REQUIRE(x && y && saved, HK_ERR_ARG, "hk_sqrtm_fwd: null pointer");
  HK_REQUIRE(iterN >= 2, HK_ERR_UNSUPPORTED, "hk_sqrtm_fwd: iterN=%d (< 2) is not supported", iterN);
  HK_REQUIRE(n % 4 == 0, HK_ERR_UNSUPPORTED, "hk_sqrtm_fwd: dim=%d must be a multiple of 4", n);
  HK_REQUIRE(workspace && workspace_bytes >= hk_sqrtm_fwd_workspace_bytes(B, n), HK_ERR_WORKSPACE,
             "hk_sqrtm_fwd: workspace too small");
  SqrtmSaved sv = saved_view(saved, B, n, iterN);
  const size_t S = sv.S;
  const int L = sv.L;
  float* w = static_cast<float*>(workspace);       // matrix slot 0 is unused
  Pair ZY = {w + S, w + 2 * S};
  Pair T = {w + 3 * S, w + 4 * S};
  int r;
  trace_normalize_kernel<<<B, 256, 0, st>>>(x, sv.normA, sv.A.hi, sv.A.lo, n);
  HK_LAUNCH_CHECK("trace_normalize_kernel");
  // ZY = 0.5 (3I - A) ; Z_0 = ZY ; Y_0 = A . ZY                                     (MPNCOV.py:153-155)
  affine_diag_split_kernel<<<grid_1d(S, 256), 256, 0, st>>>(sv.A.hi, sv.A.lo, sv.Z(0).hi, sv.Z(0).lo, -0.5f, nullptr, 0,
                                                            1.5f, n, S);
  HK_LAUNCH_CHECK("affine_diag_split_kernel");
  if ((r = mm3(sv.A, sv.Z(0), sv.Y(0), n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
  for (int i = 1; i < L; ++i) {                                                   // (MPNCOV.py:156-159)
    if ((r = mm3(sv.Z(i - 1), sv.Y(i - 1), ZY, n, B, -0.5f, 1.5f, nullptr, 0.f, st))) return r;
    if ((r = mm3(sv.Y(i - 1), ZY, sv.Y(i), n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
    if ((r = mm3(ZY, sv.Z(i - 1), sv.Z(i), n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
  }
  // YZY = 0.5 Y (3I - Z Y) ; y = YZY sqrt(normA)                                   (MPNCOV.py:160-161)
  if ((r = mm3(sv.Z(L - 1), sv.Y(L - 1), T, n, B, -1.f, 3.f, nullptr, 0.f, st))) return r;
  if ((r = mm3(sv.Y(L - 1), T, ZY, n, B, 0.5f, 0.f, nullptr, 0.f, st))) return r;
  pair_combine_scale_kernel<<<grid_1d(S, 256), 256, 0, st>>>(ZY.hi, ZY.lo, y, sv.normA, 1, (size_t)n * n, S);
  HK_LAUNCH_CHECK("pair_combine_scale_kernel");
  return 0;
}

/* Sqrtm.backward (MPNCOV.py:166-202), the reference's formulae in the reference's operand order.
 * x = forward input, y = forward output, g = grad_output, saved = what hk_sqrtm_fwd wrote. */
int hk_sqrtm_bwd(const float* x, const float* y, const float* g, float* saved, float* grad_x, int B, int n, int iterN,
                 void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  HK_REQUIRE(x && y && g && saved && grad_x, HK_ERR_ARG, "hk_sqrtm_bwd: null pointer");
  HK_REQUIRE(iterN >= 2, HK_ERR_UNSUPPORTED, "hk_sqrtm_bwd: iterN=%d (< 2) is not supported", iterN);
  HK_REQUIRE(n % 4 == 0, HK_ERR_UNSUPPORTED, "hk_sqrtm_bwd: dim=%d must be a multiple of 4", n);
  HK_REQUIRE(workspace && workspace_bytes >= hk_sqrtm_bwd_workspace_bytes(B, n), HK_ERR_WORKSPACE,
             "hk_sqrtm_bwd: workspace too small");
  SqrtmSaved sv = saved_view(saved, B, n, iterN);
  const size_t S = sv.S;
  const int L = sv.L;
  float* w = static_cast<float*>(workspace);
  int slot = 1;                                      // matrix slot 0 is unused
  auto newp = [&]() { Pair p{w + (size_t)slot * S, w + (size_t)(slot + 1) * S}; slot += 2; return p; };
  Pair P = newp(), T1 = newp(), U = newp(), V = newp(), dY = newp(), dZ = newp(), W2 = newp(), dY2 = newp(), dZ2 = newp(),
       acc = newp(), E1 = newp();   // 11 pairs = 22 matrices + slot 0 = 23
  int r;
  // der_postCom = g sqrt(normA)                                                       (MPNCOV.py:174)
  affine_diag_split_kernel<<<grid_1d(S, 256), 256, 0, st>>>(g, nullptr, P.hi, P.lo, 1.f, sv.normA, 1, 0.f, n, S);
  HK_LAUNCH_CHECK("affine_diag_split_kernel");
  const Pair Yl = sv.Y(L - 1), Zl = sv.Z(L - 1);
  // dldY = 0.5 (P (3I - Yl Zl) - Zl Yl P)                                            (MPNCOV.py:180-181)
  if ((r = mm3(Yl, Zl, T1, n, B, -1.f, 3.f, nullptr, 0.f, st))) return r;
  if ((r = mm3(P, T1, U, n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
  if ((r = mm3(Zl, Yl, V, n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
  if ((r = mm3(V, P, dY, n, B, -0.5f, 0.f, &U, 0.5f, st))) return r;
  // dldZ = -0.5 Yl P Yl                                                              (MPNCOV.py:182)
  if ((r = mm3(Yl, P, W2, n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
  if ((r = mm3(W2, Yl, dZ, n, B, -0.5f, 0.f, nullptr, 0.f, st))) return r;
  for (int i = L - 2; i >= 0; --i) {                                                // (MPNCOV.py:183-193)
    const Pair Yi = sv.Y(i), Zi = sv.Z(i);
    if ((r = mm3(Yi, Zi, T1, n, B, -1.f, 3.f, nullptr, 0.f, st))) return r;   // YZ = 3I - Y Z
    if ((r = mm3(Zi, Yi, V, n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;     // ZY = Z Y
    // dldY_ = 0.5 (dldY YZ - Z dldZ Z - ZY dldY)
    if ((r = mm3(dY, T1, U, n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
    if ((r = mm3(Zi, dZ, W2, n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
    if ((r = mm3(W2, Zi, acc, n, B, -0.5f, 0.f, &U, 0.5f, st))) return r;
    if ((r = mm3(V, dY, dY2, n, B, -0.5f, 0.f, &acc, 1.f, st))) return r;
    // dldZ_ = 0.5 (YZ dldZ - Y dldY Y - dldZ ZY)
    if ((r = mm3(T1, dZ, U, n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
    if ((r = mm3(Yi, dY, W2, n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
    if ((r = mm3(W2, Yi, acc, n, B, -0.5f, 0.f, &U, 0.5f, st))) return r;
    if ((r = mm3(dZ, V, dZ2, n, B, -0.5f, 0.f, &acc, 1.f, st))) return r;
    Pair t = dY; dY = dY2; dY2 = t;
    t = dZ; dZ = dZ2; dZ2 = t;
  }
  // der_NSiter = 0.5 (dldY (3I - A) - dldZ - A dldY)                                  (MPNCOV.py:194)
  affine_diag_split_kernel<<<grid_1d(S, 256), 256, 0, st>>>(sv.A.hi, sv.A.lo, E1.hi, E1.lo, -1.f, nullptr, 0, 3.f, n, S);
  HK_LAUNCH_CHECK("affine_diag_split_kernel");
  if ((r = mm3(dY, E1, U, n, B, 1.f, 0.f, nullptr, 0.f, st))) return r;
  if ((r = mm3(sv.A, dY, acc, n, B, -0.5f, 0.f, &U, 0.5f, st))) return r;   // acc = 0.5 dldY(3I-A) - 0.5 A dldY
  // transpose, /normA, diagonal correction                                            (MPNCOV.py:195-201)
  sqrtm_bwd_tail_kernel<<<B, 256, 0, st>>>(acc.hi, acc.lo, dZ.hi, dZ.lo, x, y, g, sv.normA, grad_x, n);
  HK_LAUNCH_CHECK("sqrtm_bwd_tail_kernel");
  return 0;
}

/* ---------------- Triuvec (MPNCOV.py:205-230) ---------------- */
int hk_triuvec_fwd(const float* x, float* y, int B, int n, void* stream) {
  HK_REQUIRE(x && y, HK_ERR_ARG, "hk_triuvec_fwd: null pointer");
  triuvec_fwd_kernel<<<dim3(n, B), 128, 0, (cudaStream_t)stream>>>(x, y, n);
  HK_LAUNCH_CHECK("triuvec_fwd_kernel");
  return 0;
}
int hk_triuvec_bwd(const float* g, float* dx, int B, int n, void* stream) {
  HK_REQUIRE(g && dx, HK_ERR_ARG, "hk_triuvec_bwd: null pointer");
  triuvec_bwd_kernel<<<dim3(n, B), 128, 0, (cudaStream_t)stream>>>(g, dx, n);
  HK_LAUNCH_CHECK("triuvec_bwd_kernel");
  return 0;
}

}  // extern "C"
