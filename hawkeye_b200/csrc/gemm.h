// Epilogue description + host entries of the generic batched wgmma TF32 GEMM and its split-K form (gemm.cu).
#pragma once
#include <cuda_runtime.h>
#include <type_traits>

namespace hk {

enum { EPI_PLAIN = 0, EPI_BILINEAR_S = 1, EPI_SKETCH = 2 };

// Every field defaults to null / zero / EPI_PLAIN; callers set the ones they use.
struct GemmEpi {
  float* C = nullptr;
  long long ldc = 0, strideC = 0;
  const float* D = nullptr;
  long long ldd = 0, strideD = 0;
  const float* alpha_vec = nullptr;
  const float* beta_vec = nullptr;
  float alpha = 0.f, beta = 0.f, diag = 0.f;
  int trans_c = 0;
  int relu = 0;                  // bit0: ReLU, bit1: round the stored value to tf32
  float* C_lo = nullptr;         // optional: store C as a (hi, lo) tf32 pair (3xTF32 operands for the next GEMM)
  const float* D_lo = nullptr;   // optional: D given as a (hi, lo) pair
  const float* E = nullptr;      // optional: raw partial product added to the accumulator before alpha (row-major [M][N] per batch)
  long long ldE = 0, strideE = 0;   // layout of E; 0 = same as C (ldc / strideC)
  const float* post_scale = nullptr;  // optional [batch]: value = sqrt(alpha_b * acc + post_eps) * post_scale[b], then D / ReLU / rounding
  float post_eps = 0.f;
  // Fused consumers of a square Gram G = alpha_b * acc (M = N = C, row-major [C][C] per batch entry):
  //   EPI_BILINEAR_S: C[i][j] = (dY[i][j] + dY[j][i]) / (2 z_ij), z_ij = sqrt(G_ij + post_eps); c_raw[b] += sum_ij dY_ij z_ij
  //                   (c_raw pre-zeroed) — the bilinear-pool backward's S without the Gram going through memory;
  //   EPI_SKETCH    : bins[b][(h1[i] + h2[j]) mod d] += s1[i] s2[j] G_ij (bins pre-zeroed); C is not written.
  int mode = EPI_PLAIN;
  const float* dY = nullptr;
  double* c_raw = nullptr;
  const int* h1 = nullptr;
  const int* h2 = nullptr;
  const float* s1 = nullptr;
  const float* s2 = nullptr;
  float* bins = nullptr;
  int d = 0;
};
static_assert(std::is_aggregate_v<GemmEpi> && std::is_trivially_copyable_v<GemmEpi>,
              "GemmEpi is passed to the GEMM kernel by value");

// C[b] = alpha_b * (A[b].B[b] + E[b]) + diag*I + beta_b * (D[b] + D_lo[b]);  see hk_gemm_tf32 in the public header.
// Dispatches on the precision mode (host.h): one TF32 pass, or 3xTF32 over internally split operands.
int gemm_tf32(const float* A, int a_mn, long long lda, long long strideA, const float* B, int b_mn, long long ldb,
              long long strideB, const GemmEpi& epi, int M, int N, int K, int batch, cudaStream_t stream);
// Always one TF32 pass (callers that manage (hi, lo) operand pairs themselves: the Newton-Schulz chain).
int gemm_tf32_1x(const float* A, int a_mn, long long lda, long long strideA, const float* B, int b_mn, long long ldb,
                 long long strideB, const GemmEpi& epi, int M, int N, int K, int batch, cudaStream_t stream);

// One launch of the 3xTF32 product for operands already held as tf32 (hi, lo) pairs:  C = epilogue(Ah.Bh + Al.Bh + Ah.Bl).
int gemm_tf32_pair(const float* Ah, const float* Al, int a_mn, long long lda, long long strideA, const float* Bh,
                   const float* Bl, int b_mn, long long ldb, long long strideB, const GemmEpi& epi, int M, int N, int K,
                   int batch, cudaStream_t stream);

// Split-K product out[M][0:cols) (+)= bias + A.B for one A [M,K] (or [K,M] if a_mn) and B [N,K] (or [K,N] if b_mn):
// an S-way batched GEMM over the K/S-long slices (S divides K) writes part [S][M][N] (the caller's workspace), which
// sum_splits reduces into out (leading dimension ldo).  With S == 1, no bias, no accumulation and out covering the
// whole product, the GEMM writes out directly.
int gemm_splitk(const float* A, int a_mn, long long lda, const float* B, int b_mn, long long ldb, int M, int N, long long K,
                int S, float* part, float* out, long long ldo, int cols, const float* bias, bool accumulate,
                cudaStream_t stream);
// out[r][c] = (accumulate ? out[r][c] : 0) + s,  s = (bias ? bias[c] : 0) + part_0[r][c] + ... + part_{S-1}[r][c], summed
// in that order; partial k starts at part + k * split_stride and its rows are ldp floats apart.
int sum_splits(const float* part, int S, long long split_stride, int rows, int cols, long long ldp, float* out,
               long long ldo, const float* bias, bool accumulate, cudaStream_t stream);

}  // namespace hk
