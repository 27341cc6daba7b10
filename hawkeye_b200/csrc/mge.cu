// MGE-CNN (reference model/methods/MGE_CNN/MGE.py, grad_cam.py): the conv6* part head (1x1 conv with padding 1, ReLU and a
// global max), the Grad-CAM box of one image in closed form, the detached 10 * l2-normalised concatenation, and the
// softmax gate over the three experts.  The reference runs a full autograd backward inside its forward for each CAM and
// builds the boxes with nonzero() and a host-side test per image (MGE.py:48-72, :145-190); nothing here leaves the device.
// Every sum runs in a fixed order (no atomics): the same bits on every run.
#include "common.cuh"
#include "gemm.h"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

constexpr int MGE_CAM_THREADS = 1024;
constexpr int MGE_GATES = 3;

// ---------------------------------------------------------------------------------------------------------------
// part head: y [N, HW, O] = x w^T + b (the wgmma GEMM) -> pooled [N, O], pos [N, O]
// ---------------------------------------------------------------------------------------------------------------
// Conv2d(1024, O, 1, 1, 1) pads the map by one pixel, where the output is its bias: relu(b_o) takes part in the max.  The
// padded map is scanned row-major from its all-border first row, so a tie between the border and the interior goes to the
// border; inside, the first maximum in row-major order wins (adaptive_max_pool2d's rule).
__global__ void mge_part_pool_kernel(const float* __restrict__ y, const float* __restrict__ bias, float* __restrict__ pooled,
                                     int* __restrict__ pos, int N, int HW, int O, int round) {
  const size_t total = (size_t)N * O;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int o = (int)(i % O), n = (int)(i / O);
    const float* col = y + (size_t)n * HW * O + o;
    float best = -INFINITY;
    int arg = 0;
    for (int p = 0; p < HW; ++p) {
      const float v = col[(size_t)p * O];
      if (v > best) { best = v; arg = p; }
    }
    const float border = fmaxf(bias[o], 0.f), inner = fmaxf(best, 0.f);
    const float v = border >= inner ? border : inner;
    pooled[i] = round ? tf32_round(v) : v;
    pos[i] = border >= inner ? -1 : arg;
  }
}

// dw[o, c] = sum_n g[n, o] [pooled[n, o] > 0] x[n, pos[n, o], c], n ascending; the border (pos -1) has no weight term
__global__ void mge_part_dw_kernel(const float* __restrict__ x, const int* __restrict__ pos, const float* __restrict__ pooled,
                                   const float* __restrict__ g, float* __restrict__ dw, int N, int HW, int C, int O) {
  const size_t total = (size_t)O * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C), o = (int)(i / C);
    float acc = 0.f;
    for (int n = 0; n < N; ++n) {
      const size_t r = (size_t)n * O + o;
      const int p = pos[r];
      if (p >= 0 && pooled[r] > 0.f) acc = fmaf(g[r], x[((size_t)n * HW + p) * C + c], acc);
    }
    dw[i] = acc;
  }
}

// db[o] = sum_n g[n, o] [pooled[n, o] > 0]: border or interior, the winner moves with b_o
__global__ void mge_part_db_kernel(const float* __restrict__ pooled, const float* __restrict__ g, float* __restrict__ db, int N,
                                   int O) {
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < O; o += gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int n = 0; n < N; ++n) {
      const size_t r = (size_t)n * O + o;
      if (pooled[r] > 0.f) acc += g[r];
    }
    db[o] = acc;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// CAM box of one image per block
// ---------------------------------------------------------------------------------------------------------------
// upsample_bilinear2d (align_corners=True) source taps of output index d, with ATen's fp32 arithmetic: src = scale d,
// i0 = min(floor(src), in - 1), lambda = clamp(src - i0, 0, 1), i1 = i0 + (i0 < in - 1)
__device__ __forceinline__ void mge_taps(float scale, int d, int in, int& i0, int& i1, float& l0, float& l1) {
  const float src = __fmul_rn(scale, (float)d);
  int i = (int)floorf(src);
  if (i > in - 1) i = in - 1;
  const float lam = fminf(fmaxf(__fsub_rn(src, (float)i), 0.f), 1.f);
  i0 = i;
  i1 = i + (i < in - 1 ? 1 : 0);
  l1 = lam;
  l0 = __fsub_rn(1.f, lam);
}

// the upsampled CAM at (oy, ox): (v00 w0 + v01 w1) h0 + (v10 w0 + v11 w1) h1, unfused, in ATen's CPU order
__device__ __forceinline__ float mge_cam_at(const float* cam, int h, int w, float rh, float rw, int oy, int ox) {
  int y0, y1, x0, x1;
  float h0, h1, w0, w1;
  mge_taps(rh, oy, h, y0, y1, h0, h1);
  mge_taps(rw, ox, w, x0, x1, w0, w1);
  const float top = __fadd_rn(__fmul_rn(cam[y0 * w + x0], w0), __fmul_rn(cam[y0 * w + x1], w1));
  const float bot = __fadd_rn(__fmul_rn(cam[y1 * w + x0], w0), __fmul_rn(cam[y1 * w + x1], w1));
  return __fadd_rn(__fmul_rn(top, h0), __fmul_rn(bot, h1));
}

__device__ __forceinline__ int block_min_int(int v, int* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) t = min(t, red[i]);
  return t;
}

// get_bbox (MGE.py:48-72) with the Grad-CAM weights of grad_cam.py in closed form: the hooked tensor is layer4's output,
// pooled and fed to the main classifier, so its gradient is W[idx, c] / HW everywhere and the weights are relu(W[idx]) / HW.
// idx is targets[n] or the first maximum of logits[n].  The CAM is summed over channels by one warp per pixel, upsampled to
// S x S, min-max normalised, and thresholded as sign(sign(m - rate) + 1), under which a NaN (constant CAM: 0 / 0) is kept.
__global__ void __launch_bounds__(MGE_CAM_THREADS)
    mge_cam_box_kernel(const float* __restrict__ logits, const long long* __restrict__ targets, const float* __restrict__ wmain,
                       const float* __restrict__ feat, int4* __restrict__ boxes, int K, int C, int h, int w, int S, float rate) {
  extern __shared__ float sm[];
  float* wgt = sm;              // [C]
  float* cam = sm + C;          // [h w]
  __shared__ float redf[32];
  __shared__ int redi[32];
  __shared__ int s_idx;
  const int n = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int HW = h * w;
  if (warp == 0) {
    int idx;
    if (targets) {
      const long long t = targets[n];
      idx = t >= 0 && t < K ? (int)t : -1;
    } else {
      const float* z = logits + (size_t)n * K;
      float best = -INFINITY;
      idx = K;
      for (int k = lane; k < K; k += 32)
        if (z[k] > best) { best = z[k]; idx = k; }
      warp_argmax(best, idx);
      if (idx >= K) idx = -1;
    }
    if (lane == 0) s_idx = idx;
  }
  __syncthreads();
  const int idx = s_idx;
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    wgt[c] = idx >= 0 ? fmaxf(wmain[(size_t)idx * C + c], 0.f) / (float)HW : 0.f;
  __syncthreads();
  const float* f = feat + (size_t)n * HW * C;
  for (int p = warp; p < HW; p += nw) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(f[(size_t)p * C + c], wgt[c], s);
    s = warp_sum(s);
    if (lane == 0) cam[p] = s;
  }
  __syncthreads();
  const float rh = S > 1 ? (float)(h - 1) / (float)(S - 1) : 0.f;
  const float rw = S > 1 ? (float)(w - 1) / (float)(S - 1) : 0.f;
  const int SS = S * S;
  float lo = INFINITY, hi = -INFINITY;
  for (int q = threadIdx.x; q < SS; q += blockDim.x) {
    const float v = mge_cam_at(cam, h, w, rh, rw, q / S, q % S);
    lo = fminf(lo, v);
    hi = fmaxf(hi, v);
  }
  lo = -block_max(-lo, redf);
  hi = block_max(hi, redf);
  const float range = __fsub_rn(hi, lo);
  int r0 = S, r1 = -1, c0 = S, c1 = -1;
  for (int q = threadIdx.x; q < SS; q += blockDim.x) {
    const int oy = q / S, ox = q - oy * S;
    const float m = __fdiv_rn(__fsub_rn(mge_cam_at(cam, h, w, rh, rw, oy, ox), lo), range);
    if (!(m < rate)) {            // m >= rate, or m is NaN
      r0 = min(r0, oy); r1 = max(r1, oy);
      c0 = min(c0, ox); c1 = max(c1, ox);
    }
  }
  r0 = block_min_int(r0, redi);
  r1 = -block_min_int(-r1, redi);
  c0 = block_min_int(c0, redi);
  c1 = -block_min_int(-c1, redi);
  if (threadIdx.x == 0) {
    // x[:, y1:y2, x1:x2] with the last kept row and column excluded; a box of zero height or width (or no kept pixel,
    // which only a rate above 1 gives) takes the whole image
    const bool whole = r1 < 0 || r0 == r1 || c0 == c1;
    boxes[n] = whole ? make_int4(0, 0, S, S) : make_int4(r0, c0, r1, c1);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// detached concatenation and the gate
// ---------------------------------------------------------------------------------------------------------------
// out[n] = (scale a[n] / ||a[n]||, scale b[n] / ||b[n]||): l2_norm_v2 (MGE.py:11-15) has no epsilon.  One block per row.
__global__ void mge_cat_l2n_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int Da,
                                   int Db, float scale, int round) {
  __shared__ float red[32];
  const int n = blockIdx.x;
  const float* ra = a + (size_t)n * Da;
  const float* rb = b + (size_t)n * Db;
  float* o = out + (size_t)n * (Da + Db);
  float sa = 0.f, sb = 0.f;
  for (int i = threadIdx.x; i < Da; i += blockDim.x) sa = fmaf(ra[i], ra[i], sa);
  for (int i = threadIdx.x; i < Db; i += blockDim.x) sb = fmaf(rb[i], rb[i], sb);
  const float na = sqrtf(block_sum(sa, red)), nb = sqrtf(block_sum(sb, red));
  for (int i = threadIdx.x; i < Da; i += blockDim.x) {
    const float v = __fmul_rn(__fdiv_rn(ra[i], na), scale);
    o[i] = round ? tf32_round(v) : v;
  }
  for (int i = threadIdx.x; i < Db; i += blockDim.x) {
    const float v = __fmul_rn(__fdiv_rn(rb[i], nb), scale);
    o[Da + i] = round ? tf32_round(v) : v;
  }
}

// One warp per image: z = h w2^T + b2, pr = softmax(z), out[n, k] = (c0 pr0 + c1 pr1) + c2 pr2 (MGE.py:207-213)
__global__ void mge_gate_fwd_kernel(const float* __restrict__ hid, const float* __restrict__ w2, const float* __restrict__ b2,
                                    const float* __restrict__ c0, const float* __restrict__ c1, const float* __restrict__ c2,
                                    float* __restrict__ pr, float* __restrict__ out, int N, int F, int K) {
  const int lane = threadIdx.x & 31;
  const int n = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
  if (n >= N) return;
  const float* hr = hid + (size_t)n * F;
  float z[MGE_GATES];
#pragma unroll
  for (int j = 0; j < MGE_GATES; ++j) {
    float s = 0.f;
    for (int f = lane; f < F; f += 32) s = fmaf(hr[f], w2[(size_t)j * F + f], s);
    z[j] = warp_sum(s) + b2[j];
  }
  const float m = fmaxf(fmaxf(z[0], z[1]), z[2]);
  const float e0 = expf(z[0] - m), e1 = expf(z[1] - m), e2 = expf(z[2] - m);
  const float se = (e0 + e1) + e2;
  const float p0 = e0 / se, p1 = e1 / se, p2 = e2 / se;
  if (lane == 0) {
    pr[(size_t)n * 3] = p0;
    pr[(size_t)n * 3 + 1] = p1;
    pr[(size_t)n * 3 + 2] = p2;
  }
  const size_t r = (size_t)n * K;
  for (int k = lane; k < K; k += 32)
    out[r + k] = __fadd_rn(__fadd_rn(__fmul_rn(c0[r + k], p0), __fmul_rn(c1[r + k], p1)), __fmul_rn(c2[r + k], p2));
}

// One warp per image: d_j = <dout[n], c_j[n]> (+ dpr[n, j]), dz_j = pr_j (d_j - sum_i pr_i d_i), dh[n] = dz w2
__global__ void mge_gate_bwd_rows_kernel(const float* __restrict__ w2, const float* __restrict__ pr, const float* __restrict__ c0,
                                         const float* __restrict__ c1, const float* __restrict__ c2, const float* __restrict__ dout,
                                         const float* __restrict__ dpr, float* __restrict__ dz, float* __restrict__ dh, int N,
                                         int F, int K) {
  const int lane = threadIdx.x & 31;
  const int n = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
  if (n >= N) return;
  const size_t r = (size_t)n * K;
  float d0 = 0.f, d1 = 0.f, d2 = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float g = dout[r + k];
    d0 = fmaf(g, c0[r + k], d0);
    d1 = fmaf(g, c1[r + k], d1);
    d2 = fmaf(g, c2[r + k], d2);
  }
  d0 = warp_sum(d0);
  d1 = warp_sum(d1);
  d2 = warp_sum(d2);
  if (dpr) {
    d0 += dpr[(size_t)n * 3];
    d1 += dpr[(size_t)n * 3 + 1];
    d2 += dpr[(size_t)n * 3 + 2];
  }
  const float p0 = pr[(size_t)n * 3], p1 = pr[(size_t)n * 3 + 1], p2 = pr[(size_t)n * 3 + 2];
  const float s = (p0 * d0 + p1 * d1) + p2 * d2;
  const float z0 = p0 * (d0 - s), z1 = p1 * (d1 - s), z2 = p2 * (d2 - s);
  if (lane == 0) {
    dz[(size_t)n * 3] = z0;
    dz[(size_t)n * 3 + 1] = z1;
    dz[(size_t)n * 3 + 2] = z2;
  }
  if (dh)
    for (int f = lane; f < F; f += 32)
      dh[(size_t)n * F + f] = fmaf(z2, w2[2 * (size_t)F + f], fmaf(z1, w2[(size_t)F + f], z0 * w2[f]));
}

// dw2[j, f] = sum_n dz[n, j] h[n, f], db2[j] = sum_n dz[n, j], n ascending
__global__ void mge_gate_bwd_params_kernel(const float* __restrict__ hid, const float* __restrict__ dz, float* __restrict__ dw2,
                                           float* __restrict__ db2, int N, int F) {
  const int total = MGE_GATES * (F + 1);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int j = i / (F + 1), f = i - j * (F + 1);
    float acc = 0.f;
    if (f < F) {
      for (int n = 0; n < N; ++n) acc = fmaf(dz[(size_t)n * 3 + j], hid[(size_t)n * F + f], acc);
      dw2[(size_t)j * F + f] = acc;
    } else {
      for (int n = 0; n < N; ++n) acc += dz[(size_t)n * 3 + j];
      db2[j] = acc;
    }
  }
}

}  // namespace hk

using namespace hk;

extern "C" {

size_t hk_mge_part_workspace_bytes(int N, int H, int W, int O) {
  if (N <= 0 || H <= 0 || W <= 0 || O <= 0) return 0;
  return (size_t)N * H * W * O * sizeof(float);
}

int hk_mge_part_fwd(const float* x, const float* w, const float* bias, float* pooled, int* pos, int N, int H, int W, int C,
                    int O, void* workspace, size_t workspace_bytes, void* stream) {
  HK_REQUIRE(x && w && bias && pooled && pos, HK_ERR_ARG, "hk_mge_part_fwd: null pointer");
  HK_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && O > 0 && (long long)N * H * W <= (1ll << 30), HK_ERR_ARG,
             "hk_mge_part_fwd: N=%d H=%d W=%d C=%d O=%d", N, H, W, C, O);
  HK_REQUIRE(C % 4 == 0 && O % 4 == 0, HK_ERR_UNSUPPORTED, "hk_mge_part_fwd: C=%d and O=%d must be multiples of 4", C, O);
  HK_REQUIRE(workspace && workspace_bytes >= hk_mge_part_workspace_bytes(N, H, W, O), HK_ERR_WORKSPACE,
             "hk_mge_part_fwd: workspace too small");
  HK_REQUIRE(aligned16(x) && aligned16(w) && aligned16(workspace), HK_ERR_ALIGN, "hk_mge_part_fwd: unaligned pointer");
  float* y = static_cast<float*>(workspace);
  GemmEpi e = {};
  e.C = y; e.ldc = O; e.alpha = 1.f;
  e.D = bias; e.ldd = 0; e.beta = 1.f;          // ldd 0: the bias row is added to every pixel
  const int P = N * H * W;
  if (int r = gemm_tf32(x, 0, C, 0, w, 0, C, 0, e, P, O, C, 1, (cudaStream_t)stream)) return r;
  mge_part_pool_kernel<<<grid_1d((size_t)N * O, 256), 256, 0, (cudaStream_t)stream>>>(y, bias, pooled, pos, N, H * W, O,
                                                                                     precise() ? 0 : 1);
  HK_LAUNCH_CHECK("mge_part_pool_kernel");
  return 0;
}

int hk_mge_part_bwd(const float* x, const int* pos, const float* pooled, const float* dpooled, float* dw, float* db, int N,
                    int H, int W, int C, int O, void* stream) {
  HK_REQUIRE(x && pos && pooled && dpooled && dw && db, HK_ERR_ARG, "hk_mge_part_bwd: null pointer");
  HK_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && O > 0, HK_ERR_ARG, "hk_mge_part_bwd: N=%d H=%d W=%d C=%d O=%d", N, H, W,
             C, O);
  mge_part_dw_kernel<<<grid_1d((size_t)O * C, 256), 256, 0, (cudaStream_t)stream>>>(x, pos, pooled, dpooled, dw, N, H * W, C,
                                                                                    O);
  HK_LAUNCH_CHECK("mge_part_dw_kernel");
  mge_part_db_kernel<<<grid_1d((size_t)O, 256), 256, 0, (cudaStream_t)stream>>>(pooled, dpooled, db, N, O);
  HK_LAUNCH_CHECK("mge_part_db_kernel");
  return 0;
}

int hk_mge_cam_box(const float* logits, const long long* targets, const float* w_main, const float* feat, int* boxes, int N,
                   int K, int C, int h, int w, int S, float rate, void* stream) {
  HK_REQUIRE((logits || targets) && w_main && feat && boxes, HK_ERR_ARG, "hk_mge_cam_box: null pointer");
  HK_REQUIRE(N > 0 && K > 0 && C > 0 && h > 0 && w > 0 && S > 1, HK_ERR_ARG, "hk_mge_cam_box: N=%d K=%d C=%d h=%d w=%d S=%d",
             N, K, C, h, w, S);
  HK_REQUIRE(N <= 65535 && (long long)S * S <= (1ll << 30), HK_ERR_ARG, "hk_mge_cam_box: N=%d S=%d", N, S);
  const size_t smem = ((size_t)C + (size_t)h * w) * sizeof(float);
  HK_REQUIRE(smem <= 48 * 1024, HK_ERR_UNSUPPORTED, "hk_mge_cam_box: C + h w = %zu floats, at most 12288", smem / 4);
  HK_REQUIRE(aligned16(boxes), HK_ERR_ALIGN, "hk_mge_cam_box: boxes must be 16-byte aligned");
  mge_cam_box_kernel<<<N, MGE_CAM_THREADS, smem, (cudaStream_t)stream>>>(targets ? nullptr : logits, targets, w_main, feat,
                                                                        reinterpret_cast<int4*>(boxes), K, C, h, w, S, rate);
  HK_LAUNCH_CHECK("mge_cam_box_kernel");
  return 0;
}

int hk_mge_cat_l2n(const float* a, const float* b, float* out, int N, int Da, int Db, float scale, void* stream) {
  HK_REQUIRE(a && b && out, HK_ERR_ARG, "hk_mge_cat_l2n: null pointer");
  HK_REQUIRE(N > 0 && N <= 65535 && Da > 0 && Db > 0, HK_ERR_ARG, "hk_mge_cat_l2n: N=%d Da=%d Db=%d", N, Da, Db);
  mge_cat_l2n_kernel<<<N, 256, 0, (cudaStream_t)stream>>>(a, b, out, Da, Db, scale, precise() ? 0 : 1);
  HK_LAUNCH_CHECK("mge_cat_l2n_kernel");
  return 0;
}

int hk_mge_gate_fwd(const float* h, const float* w2, const float* b2, const float* c0, const float* c1, const float* c2,
                    float* pr, float* out, int N, int F, int K, void* stream) {
  HK_REQUIRE(h && w2 && b2 && c0 && c1 && c2 && pr && out, HK_ERR_ARG, "hk_mge_gate_fwd: null pointer");
  HK_REQUIRE(N > 0 && F > 0 && K > 0, HK_ERR_ARG, "hk_mge_gate_fwd: N=%d F=%d K=%d", N, F, K);
  mge_gate_fwd_kernel<<<grid_1d((size_t)N * 32, 256), 256, 0, (cudaStream_t)stream>>>(h, w2, b2, c0, c1, c2, pr, out, N, F, K);
  HK_LAUNCH_CHECK("mge_gate_fwd_kernel");
  return 0;
}

int hk_mge_gate_bwd(const float* h, const float* w2, const float* pr, const float* c0, const float* c1, const float* c2,
                    const float* dout, const float* dpr, float* dz, float* dh, float* dw2, float* db2, int N, int F, int K,
                    void* stream) {
  HK_REQUIRE(h && w2 && pr && c0 && c1 && c2 && dout && dz, HK_ERR_ARG, "hk_mge_gate_bwd: null pointer");
  HK_REQUIRE(!dw2 == !db2, HK_ERR_ARG, "hk_mge_gate_bwd: dw2 and db2 go together");
  HK_REQUIRE(N > 0 && F > 0 && K > 0, HK_ERR_ARG, "hk_mge_gate_bwd: N=%d F=%d K=%d", N, F, K);
  mge_gate_bwd_rows_kernel<<<grid_1d((size_t)N * 32, 256), 256, 0, (cudaStream_t)stream>>>(w2, pr, c0, c1, c2, dout, dpr, dz,
                                                                                          dh, N, F, K);
  HK_LAUNCH_CHECK("mge_gate_bwd_rows_kernel");
  if (dw2) {
    mge_gate_bwd_params_kernel<<<grid_1d((size_t)MGE_GATES * (F + 1), 256), 256, 0, (cudaStream_t)stream>>>(h, dz, dw2, db2, N,
                                                                                                           F);
    HK_LAUNCH_CHECK("mge_gate_bwd_params_kernel");
  }
  return 0;
}

}  // extern "C"
