// NTS-Net (reference model/methods/NTS_Net/NTSNet.py, anchors.py, model/loss/NTS_loss.py): the navigator's scoring head,
// the greedy NMS with the gather of the kept scores, the part crops, and the ranking loss, all on the device.  The reference
// copies the scores to the host for a numpy NMS (NTSNet.py:33-38), crops with B x topN separate F.interpolate calls
// (:40-48) and reads every label back in list_loss (NTS_loss.py:32-35); nothing here leaves the device.  down1..3 run on
// hk_conv3x3_*, the classifiers on hk_linear_*, the cross-entropies on hk_softmax_ce_ls.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

constexpr int NTS_MAX_ANCHORS = 2048;     // NMS keeps scores, boxes and the alive flags of one image in shared memory
constexpr int NTS_TIDY = 21;              // 6 + 6 + 9 tidy outputs
constexpr int NTS_NMS_THREADS = 512;

struct TidyMaps {
  const float* d[3];
  const float* w[3];
  const float* b[3];
  int hw[3];
  int na[3];        // anchors per position: 6, 6, 9
  int off[3];       // first score of each segment
};

// score index a of an image -> (segment k, tidy channel ch, position p); a = off[k] + ch * hw[k] + p (view(B, -1) of the
// NCHW tidy output, NTSNet.py:79-82)
__device__ __forceinline__ int tidy_locate(const TidyMaps& m, int a, int& ch, int& p) {
  const int k = a < m.off[1] ? 0 : (a < m.off[2] ? 1 : 2);
  const int r = a - m.off[k];
  ch = r / m.hw[k];
  p = r - ch * m.hw[k];
  return k;
}

// One warp per score: the 1x1 conv of one tidy channel at one position, lane-strided over C, the fixed xor tree, + bias.
__global__ void nts_score_fwd_kernel(TidyMaps m, float* __restrict__ score, int B, int A, int C) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long i = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); i < (long long)B * A; i += nwarps) {
    const int n = (int)(i / A), a = (int)(i - (long long)n * A);
    int ch, p;
    const int k = tidy_locate(m, a, ch, p);
    const float* x = m.d[k] + ((size_t)n * m.hw[k] + p) * C;
    const float* w = m.w[k] + (size_t)ch * C;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(x[c], w[c], s);
    s = warp_sum(s);
    if (lane == 0) score[i] = s + m.b[k][ch];
  }
}

// g_k [B, HW_k, C] = (d_k > 0) * sum over the kept scores t of image n at (k, ., p) of dprob[n, t] w_k[ch, c]: the gradient
// at the pre-activation of down_k from the tidy path.  Only the T kept scores of an image are non-zero, so each element
// scans those T entries (ascending t) instead of a dense [B, A] gradient.
__global__ void nts_score_bwd_maps_kernel(TidyMaps m, const long long* __restrict__ idx, const float* __restrict__ dprob,
                                          float* __restrict__ g0, float* __restrict__ g1, float* __restrict__ g2, int B, int A,
                                          int T, int C) {
  const long long n0 = (long long)B * m.hw[0] * C, n1 = (long long)B * m.hw[1] * C, n2 = (long long)B * m.hw[2] * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n0 + n1 + n2; i += (long long)gridDim.x * blockDim.x) {
    int k;
    long long j;
    float* g;
    if (i < n0) { k = 0; j = i; g = g0; }
    else if (i < n0 + n1) { k = 1; j = i - n0; g = g1; }
    else { k = 2; j = i - n0 - n1; g = g2; }
    const int c = (int)(j % C);
    const long long np = j / C;
    const int n = (int)(np / m.hw[k]), p = (int)(np - (long long)n * m.hw[k]);
    float s = 0.f;
    for (int t = 0; t < T; ++t) {
      const long long a = idx[(size_t)n * T + t];
      if (a < 0 || a >= A) continue;
      int ch, pp;
      if (tidy_locate(m, (int)a, ch, pp) != k || pp != p) continue;
      s = fmaf(dprob[(size_t)n * T + t], m.w[k][(size_t)ch * C + c], s);
    }
    g[j] = m.d[k][j] > 0.f ? s : 0.f;
  }
}

// dW_k[ch, c] = sum_n sum_t dprob[n, t] d_k[n, p, c] over the kept scores at (k, ch, p), and db_k[ch] (column c == C) the
// sum of those dprob; one thread per output, ascending (n, t): the same bits on every run.
__global__ void nts_score_bwd_params_kernel(TidyMaps m, const long long* __restrict__ idx, const float* __restrict__ dprob,
                                            float* dw0, float* db0, float* dw1, float* db1, float* dw2, float* db2, int B, int A,
                                            int T, int C) {
  const int total = NTS_TIDY * (C + 1);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int row = i / (C + 1), c = i - row * (C + 1);
    const int k = row < m.na[0] ? 0 : (row < m.na[0] + m.na[1] ? 1 : 2);
    const int ch = row - (k == 0 ? 0 : (k == 1 ? m.na[0] : m.na[0] + m.na[1]));
    float s = 0.f;
    for (int n = 0; n < B; ++n)
      for (int t = 0; t < T; ++t) {
        const long long a = idx[(size_t)n * T + t];
        if (a < 0 || a >= A) continue;
        int cc, p;
        if (tidy_locate(m, (int)a, cc, p) != k || cc != ch) continue;
        const float g = dprob[(size_t)n * T + t];
        s = c == C ? s + g : fmaf(g, m.d[k][((size_t)n * m.hw[k] + p) * C + c], s);
      }
    float* dw = k == 0 ? dw0 : (k == 1 ? dw1 : dw2);
    float* db = k == 0 ? db0 : (k == 1 ? db1 : db2);
    if (c == C) db[ch] = s;
    else dw[(size_t)ch * C + c] = s;
  }
}

// keep the candidate j after a pick i iff IoU < 0.25, tested exactly on the integer boxes as 4 inter < union (hard_nms,
// anchors.py:81-88: a negative overlap extent in either dimension gives inter = 0)
__device__ __forceinline__ bool nts_suppressed(int4 a, int4 b) {
  const int dy = min(a.z, b.z) - max(a.x, b.x), dx = min(a.w, b.w) - max(a.y, b.y);
  const long long inter = (dy < 0 || dx < 0) ? 0ll : (long long)dy * dx;
  const long long uni = (long long)(a.z - a.x) * (a.w - a.y) + (long long)(b.z - b.x) * (b.w - b.y) - inter;
  return 4 * inter >= uni;
}

// One block per image: T rounds of (block argmax over the alive candidates by (score descending, index ascending), then
// suppress every alive candidate the pick covers, the pick itself included).  The same picks as sorting once and scanning.
__global__ void nts_nms_kernel(const float* __restrict__ scores, const int4* __restrict__ anchors, long long* __restrict__ idx,
                               float* __restrict__ prob, int4* __restrict__ boxes, int A, int T) {
  extern __shared__ unsigned char sm_raw[];
  int4* box = reinterpret_cast<int4*>(sm_raw);
  float* sc = reinterpret_cast<float*>(box + A);
  unsigned char* alive = reinterpret_cast<unsigned char*>(sc + A);
  __shared__ float red_v[32];
  __shared__ int red_i[32];
  __shared__ int s_pick;
  const int n = blockIdx.x;
  const float* srow = scores + (size_t)n * A;
  for (int a = threadIdx.x; a < A; a += blockDim.x) {
    box[a] = anchors[a];
    sc[a] = srow[a];
    alive[a] = 1;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int t = 0; t < T; ++t) {
    float best = -INFINITY;
    int bi = -1;
    for (int a = threadIdx.x; a < A; a += blockDim.x)
      if (alive[a] && (bi < 0 || sc[a] > best)) { best = sc[a]; bi = a; }       // ascending a: the lowest index on ties
    if (bi < 0) bi = 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi != 0x7fffffff && (bi == 0x7fffffff || ob > best || (ob == best && oi < bi))) { best = ob; bi = oi; }
    }
    if (lane == 0) { red_v[warp] = best; red_i[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float v = red_v[0];
      int b = red_i[0];
      for (int w = 1; w < nw; ++w)
        if (red_i[w] != 0x7fffffff && (b == 0x7fffffff || red_v[w] > v || (red_v[w] == v && red_i[w] < b))) {
          v = red_v[w];
          b = red_i[w];
        }
      s_pick = b;
      const size_t o = (size_t)n * T + t;
      // no candidate left: T is above the survivor bound NTSNet checks at construction; the row is marked, not guessed
      idx[o] = b == 0x7fffffff ? -1 : b;
      prob[o] = b == 0x7fffffff ? 0.f : sc[b];
      boxes[o] = b == 0x7fffffff ? make_int4(0, 0, 1, 1) : box[b];
    }
    __syncthreads();
    const int pick = s_pick;
    if (pick != 0x7fffffff) {
      const int4 pb = box[pick];
      for (int a = threadIdx.x; a < A; a += blockDim.x)
        if (alive[a] && nts_suppressed(pb, box[a])) alive[a] = 0;
    }
    __syncthreads();
  }
}

// out[r, c, oy, ox] = F.interpolate(pad(img)[n, c, y0:y1, x0:x1], (S, S), bilinear, align_corners=True) with ATen's
// upsample_bilinear2d arithmetic: fp32 scale (in - 1) / (S - 1), src = scale dst, h1 = (int)src, lambdas src - h1 and
// 1 - that, h1p = (h1 < in - 1).  Padded pixels read as zero, so no padded copy of the image exists.
__global__ void nts_crop_kernel(const float* __restrict__ img, const int4* __restrict__ boxes, float* __restrict__ out, int T,
                                int C, int H, int W, int pad, int S) {
  const int r = blockIdx.y, n = r / T;        // one grid row per part image
  const int4 bx = boxes[r];
  const int ih = bx.z - bx.x, iw = bx.w - bx.y;
  const float rh = S > 1 ? (float)(ih - 1) / (float)(S - 1) : 0.f;
  const float rw = S > 1 ? (float)(iw - 1) / (float)(S - 1) : 0.f;
  const float* src = img + (size_t)n * C * H * W;
  float* dst = out + (size_t)r * C * S * S;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < C * S * S; i += gridDim.x * blockDim.x) {
    const int c = i / (S * S), q = i - c * S * S, oy = q / S, ox = q - oy * S;
    const float h1r = rh * (float)oy;
    const int h1 = (int)h1r;
    const int h1p = h1 < ih - 1 ? 1 : 0;
    const float h1l = h1r - (float)h1, h0l = 1.f - h1l;
    const float w1r = rw * (float)ox;
    const int w1 = (int)w1r;
    const int w1p = w1 < iw - 1 ? 1 : 0;
    const float w1l = w1r - (float)w1, w0l = 1.f - w1l;
    const float* plane = src + (size_t)c * H * W;
    const int ya = bx.x + h1 - pad, yb = ya + h1p, xa = bx.y + w1 - pad, xb = xa + w1p;
    const bool ya_in = ya >= 0 && ya < H, yb_in = yb >= 0 && yb < H, xa_in = xa >= 0 && xa < W, xb_in = xb >= 0 && xb < W;
    const float v00 = ya_in && xa_in ? plane[(size_t)ya * W + xa] : 0.f;
    const float v01 = ya_in && xb_in ? plane[(size_t)ya * W + xb] : 0.f;
    const float v10 = yb_in && xa_in ? plane[(size_t)yb * W + xa] : 0.f;
    const float v11 = yb_in && xb_in ? plane[(size_t)yb * W + xb] : 0.f;
    dst[i] = h0l * (w0l * v00 + w1l * v01) + h1l * (w0l * v10 + w1l * v11);
  }
}

// One block.  nll[r] = lse(z_r) - z_r[y] (list_loss, NTS_loss.py:32-35) by one warp per row into shared memory; then one
// thread per (image n, pivot i) sums relu(1 - s_i + s_j) [L_j > L_i] over j (ranking_loss, :38-47) and another pass gives
// each score its gradient: + over pivots i it beats, - over the j that beat it, where the hinge is open (torch's relu passes
// no gradient at 0).  Sums in ascending order, the block total in fp64 in warp order.
__global__ void nts_rank_loss_kernel(const float* __restrict__ logits, const long long* __restrict__ labels,
                                     const float* __restrict__ prob, double* __restrict__ loss_acc, float* __restrict__ dprob,
                                     int B, int T, int K) {
  extern __shared__ float nll[];
  __shared__ double red[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int R = B * T;
  for (int r = warp; r < R; r += nw) {
    const float* z = logits + (size_t)r * K;
    float m = -INFINITY;
    for (int k = lane; k < K; k += 32) m = fmaxf(m, z[k]);
    m = warp_max(m);
    float se = 0.f;
    for (int k = lane; k < K; k += 32) se += expf(z[k] - m);
    se = warp_sum(se);
    if (lane == 0) {
      const long long y = labels[r / T];
      nll[r] = (m + logf(se)) - (y >= 0 && y < K ? z[y] : m + logf(se));
    }
  }
  __syncthreads();
  const float inv_b = 1.f / (float)B;
  double part = 0.0;
  for (int r = threadIdx.x; r < R; r += blockDim.x) {
    const int n = r / T, i = r - n * T;
    const float* s = prob + (size_t)n * T;
    const float* L = nll + (size_t)n * T;
    float acc = 0.f, g = 0.f;
    for (int j = 0; j < T; ++j) {
      const float h = 1.f - s[i] + s[j];
      if (L[j] > L[i] && h > 0.f) { acc += h; g -= inv_b; }    // i as the pivot: d/ds_i = -1
      const float h2 = 1.f - s[j] + s[i];
      if (L[i] > L[j] && h2 > 0.f) g += inv_b;                  // i as the j of pivot j: d/ds_i = +1
    }
    part += (double)acc;
    dprob[r] = g;
  }
  const double tot = block_sum(part, red);
  if (threadIdx.x == 0) loss_acc[0] += tot / (double)B;
}

static int tidy_maps(TidyMaps& m, const float* d1, const float* d2, const float* d3, const float* w1, const float* b1,
                     const float* w2, const float* b2, const float* w3, const float* b3, int H1, int W1, int H2, int W2, int H3,
                     int W3, const char* op) {
  HK_REQUIRE(H1 > 0 && W1 > 0 && H2 == (H1 + 1) / 2 && W2 == (W1 + 1) / 2 && H3 == (H2 + 1) / 2 && W3 == (W2 + 1) / 2,
             HK_ERR_ARG, "%s: maps %dx%d, %dx%d, %dx%d are not a stride-2 (ceil) chain", op, H1, W1, H2, W2, H3, W3);
  m.d[0] = d1; m.d[1] = d2; m.d[2] = d3;
  m.w[0] = w1; m.w[1] = w2; m.w[2] = w3;
  m.b[0] = b1; m.b[1] = b2; m.b[2] = b3;
  m.hw[0] = H1 * W1; m.hw[1] = H2 * W2; m.hw[2] = H3 * W3;
  m.na[0] = 6; m.na[1] = 6; m.na[2] = 9;
  m.off[0] = 0; m.off[1] = 6 * m.hw[0]; m.off[2] = m.off[1] + 6 * m.hw[1];
  return 0;
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_nts_num_anchors(int H1, int W1) {
  if (H1 <= 0 || W1 <= 0) return 0;
  const int H2 = (H1 + 1) / 2, W2 = (W1 + 1) / 2, H3 = (H2 + 1) / 2, W3 = (W2 + 1) / 2;
  return 6 * H1 * W1 + 6 * H2 * W2 + 9 * H3 * W3;
}

int hk_nts_score_fwd(const float* d1, const float* d2, const float* d3, const float* w1, const float* b1, const float* w2,
                     const float* b2, const float* w3, const float* b3, float* score, int B, int H1, int W1, int H2, int W2,
                     int H3, int W3, int C, void* stream) {
  HK_REQUIRE(d1 && d2 && d3 && w1 && b1 && w2 && b2 && w3 && b3 && score, HK_ERR_ARG, "hk_nts_score_fwd: null pointer");
  HK_REQUIRE(B > 0 && C > 0, HK_ERR_ARG, "hk_nts_score_fwd: B=%d C=%d", B, C);
  TidyMaps m;
  if (int r = tidy_maps(m, d1, d2, d3, w1, b1, w2, b2, w3, b3, H1, W1, H2, W2, H3, W3, "hk_nts_score_fwd")) return r;
  const int A = hk_nts_num_anchors(H1, W1);
  nts_score_fwd_kernel<<<grid_1d((size_t)B * A * 32, 256), 256, 0, (cudaStream_t)stream>>>(m, score, B, A, C);
  HK_LAUNCH_CHECK("nts_score_fwd_kernel");
  return 0;
}

int hk_nts_score_bwd(const float* d1, const float* d2, const float* d3, const float* w1, const float* w2, const float* w3,
                     const long long* idx, const float* dprob, float* g1, float* g2, float* g3, float* dw1, float* db1,
                     float* dw2, float* db2, float* dw3, float* db3, int B, int T, int H1, int W1, int H2, int W2, int H3,
                     int W3, int C, void* stream) {
  HK_REQUIRE(d1 && d2 && d3 && w1 && w2 && w3 && idx && dprob && g1 && g2 && g3 && dw1 && db1 && dw2 && db2 && dw3 && db3,
             HK_ERR_ARG, "hk_nts_score_bwd: null pointer");
  HK_REQUIRE(B > 0 && T > 0 && C > 0, HK_ERR_ARG, "hk_nts_score_bwd: B=%d T=%d C=%d", B, T, C);
  TidyMaps m;
  // the biases are not read by the backward; any non-null pointer fills the slots
  if (int r = tidy_maps(m, d1, d2, d3, w1, w1, w2, w2, w3, w3, H1, W1, H2, W2, H3, W3, "hk_nts_score_bwd")) return r;
  const int A = hk_nts_num_anchors(H1, W1);
  const size_t nmap = (size_t)B * (m.hw[0] + m.hw[1] + m.hw[2]) * C;
  nts_score_bwd_maps_kernel<<<grid_1d(nmap, 256), 256, 0, (cudaStream_t)stream>>>(m, idx, dprob, g1, g2, g3, B, A, T, C);
  HK_LAUNCH_CHECK("nts_score_bwd_maps_kernel");
  nts_score_bwd_params_kernel<<<grid_1d((size_t)NTS_TIDY * (C + 1), 128), 128, 0, (cudaStream_t)stream>>>(
      m, idx, dprob, dw1, db1, dw2, db2, dw3, db3, B, A, T, C);
  HK_LAUNCH_CHECK("nts_score_bwd_params_kernel");
  return 0;
}

int hk_nts_nms(const float* scores, const int* anchors, long long* idx, float* prob, int* boxes, int B, int A, int T,
               void* stream) {
  HK_REQUIRE(scores && anchors && idx && prob && boxes, HK_ERR_ARG, "hk_nts_nms: null pointer");
  HK_REQUIRE(B > 0 && A > 0 && A <= NTS_MAX_ANCHORS && T > 0 && T <= A, HK_ERR_ARG, "hk_nts_nms: B=%d A=%d (<= %d) T=%d", B, A,
             NTS_MAX_ANCHORS, T);
  HK_REQUIRE(aligned16(anchors) && aligned16(boxes), HK_ERR_ALIGN, "hk_nts_nms: anchors / boxes must be 16-byte aligned");
  const size_t smem = (size_t)A * (sizeof(int4) + sizeof(float) + 1);
  nts_nms_kernel<<<B, NTS_NMS_THREADS, smem, (cudaStream_t)stream>>>(scores, reinterpret_cast<const int4*>(anchors), idx, prob,
                                                                     reinterpret_cast<int4*>(boxes), A, T);
  HK_LAUNCH_CHECK("nts_nms_kernel");
  return 0;
}

int hk_nts_crop(const float* img, const int* boxes, float* out, int B, int T, int C, int H, int W, int pad, int S,
                void* stream) {
  HK_REQUIRE(img && boxes && out, HK_ERR_ARG, "hk_nts_crop: null pointer");
  HK_REQUIRE(B > 0 && T > 0 && C > 0 && H > 0 && W > 0 && pad >= 0 && S > 0 && (long long)B * T <= 65535, HK_ERR_ARG,
             "hk_nts_crop: B=%d T=%d C=%d H=%d W=%d pad=%d S=%d", B, T, C, H, W, pad, S);
  HK_REQUIRE(aligned16(boxes), HK_ERR_ALIGN, "hk_nts_crop: boxes must be 16-byte aligned");
  const int per = C * S * S;
  const int gx = (per + 255) / 256 < 64 ? (per + 255) / 256 : 64;
  nts_crop_kernel<<<dim3(gx, B * T), 256, 0, (cudaStream_t)stream>>>(img, reinterpret_cast<const int4*>(boxes), out, T, C, H, W,
                                                                     pad, S);
  HK_LAUNCH_CHECK("nts_crop_kernel");
  return 0;
}

int hk_nts_rank_loss(const float* part_logits, const long long* labels, const float* prob, double* loss_acc, float* dprob,
                     int B, int T, int K, void* stream) {
  HK_REQUIRE(part_logits && labels && prob && loss_acc && dprob, HK_ERR_ARG, "hk_nts_rank_loss: null pointer");
  HK_REQUIRE(B > 0 && T > 0 && K > 0 && (long long)B * T <= 8192, HK_ERR_ARG, "hk_nts_rank_loss: B=%d T=%d K=%d (B T <= 8192)",
             B, T, K);
  nts_rank_loss_kernel<<<1, 1024, (size_t)B * T * sizeof(float), (cudaStream_t)stream>>>(part_logits, labels, prob, loss_acc,
                                                                                         dprob, B, T, K);
  HK_LAUNCH_CHECK("nts_rank_loss_kernel");
  return 0;
}

}  // extern "C"
