// Neural prototype trees (reference model/methods/ProtoTree/): the prototype distance with its global min-pool
// (l2conv.py:24-63, prototree.py:111-116) forward and backward, the soft decision tree (branch.py:22-57, leaf.py:30-67) as
// one routing pass per image plus its bottom-up backward, the NLL of the leaf mixture (Examples/ProtoTreeNet.py:109), and
// the derivative-free leaf update (Examples/ProtoTreeNet.py:116-132): its sum over the batch in one launch, applied in a
// second, so that data-parallel ranks can add their sums in between.
//
// Tree layout (prototree.py:271-289): a complete tree of height H, nodes numbered in pre-order (root 0, left child i + 1,
// right child i + 1 + size of the left subtree).  Branch k, the k-th branch in pre-order, uses prototype row k; leaf j is the
// j-th leaf from the left.  Inside a kernel a node is addressed by (depth d, position q) in heap order.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

constexpr int PT_MAX_HEIGHT = 12;        // 8191 nodes: the routing kernels keep one float per node in shared memory
constexpr int PT_TP = 64;                // prototypes per distance block
constexpr int PT_TH = 64;                // positions per distance tile
constexpr int PT_TD = 32;                // channels per shared-memory stage
constexpr int PT_MAX_K = 12288;          // classes: dtheta keeps one float per class in shared memory
constexpr int PT_MAX_GROUP_BYTES = 200 * 1024;   // the distance backward's per-image grouping: HW + 1 + P ints

// pre-order index of the node at depth d, heap position q (0 <= q < 2^d) of a tree of height H
__device__ __forceinline__ int pt_node(int d, int q, int H) {
  int i = 0;
  for (int t = 0; t < d; ++t) i += 1 + ((q >> (d - 1 - t)) & 1) * ((1 << (H - t)) - 1);
  return i;
}
// rank among the branches in pre-order (= prototype row) of the branch at depth d < H, position q
__device__ __forceinline__ int pt_branch(int d, int q, int H) {
  int r = 0;
  for (int t = 0; t < d; ++t) r += 1 + ((q >> (d - 1 - t)) & 1) * ((1 << (H - 1 - t)) - 1);
  return r;
}

// (max, sum of exp(theta - max)) of one leaf's parameters: softmax(theta - max(theta)) as leaf.py:67 computes it
__device__ void leaf_softmax_stats(const float* __restrict__ th, int K, float* red, float& m, float& s) {
  float v = -INFINITY;
  for (int k = threadIdx.x; k < K; k += blockDim.x) v = fmaxf(v, th[k]);
  m = block_max(v, red);
  float e = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) e += expf(th[k] - m);
  s = block_sum(e, red);
}

// Block (prototype tile, image n).  For each tile of PT_TH positions, thread (tx, ty) of a 16 x 16 grid accumulates the
// 4 x 4 squared distances sum_d (z[h, d] - p[j, d])^2 of prototypes 4 tx.. and positions 4 ty.. directly in fp32, PT_TD
// channels per shared-memory stage; the 64 x 64 distances then go through shared memory and thread j < PT_TP keeps the
// running (min, first argmin) of prototype j over the positions in row-major order.  With `act`, x is the neck's
// pre-activation: the load applies the sigmoid, and the blocks of the first prototype tile store z.
__global__ void __launch_bounds__(256) pt_dist_fwd_kernel(const float* __restrict__ x, const float* __restrict__ protos,
                                                          float* __restrict__ z, float* __restrict__ mind,
                                                          int* __restrict__ argmin, int HW, int D, int P, int act) {
  __shared__ __align__(16) float zs[PT_TD][PT_TH + 4];     // +4: 4-way instead of 32-way conflicts on the transposing store
  __shared__ __align__(16) float ps[PT_TD][PT_TP + 4];
  __shared__ float ds[PT_TH][PT_TP + 1];
  const int n = blockIdx.y, p0 = blockIdx.x * PT_TP;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const float* xn = x + (size_t)n * HW * D;
  float best = INFINITY;
  int arg = 0;
  for (int h0 = 0; h0 < HW; h0 += PT_TH) {
    float acc[4][4] = {};
    for (int d0 = 0; d0 < D; d0 += PT_TD) {
      for (int i = threadIdx.x; i < PT_TD * PT_TH; i += blockDim.x) {     // consecutive threads: consecutive channels
        const int dd = i % PT_TD, r = i / PT_TD;
        const int h = h0 + r, d = d0 + dd;
        float v = 0.f;
        if (h < HW && d < D) {
          v = xn[(size_t)h * D + d];
          if (act) {
            v = 1.f / (1.f + expf(-v));
            if (blockIdx.x == 0) z[((size_t)n * HW + h) * D + d] = v;
          }
        }
        zs[dd][r] = v;
        const int j = p0 + r;
        ps[dd][r] = (j < P && d < D) ? protos[(size_t)j * D + d] : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int dd = 0; dd < PT_TD; ++dd) {
        const float4 a = *reinterpret_cast<const float4*>(&zs[dd][4 * ty]);
        const float4 b = *reinterpret_cast<const float4*>(&ps[dd][4 * tx]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float t = av[i] - bv[j];
            acc[i][j] = fmaf(t, t, acc[i][j]);
          }
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) ds[4 * ty + i][4 * tx + j] = sqrtf(acc[i][j] + 1e-14f);
    __syncthreads();
    if (threadIdx.x < PT_TP) {
      const int hn = min(PT_TH, HW - h0);
      for (int r = 0; r < hn; ++r) {
        const float v = ds[r][threadIdx.x];
        if (v < best) { best = v; arg = h0 + r; }
      }
    }
    __syncthreads();
  }
  const int j = p0 + threadIdx.x;
  if (threadIdx.x < PT_TP && j < P) {
    mind[(size_t)n * P + j] = best;
    argmin[(size_t)n * P + j] = arg;
  }
}

// Block per image n.  Thread 0 first groups the prototypes by their argmin position (a counting sort in ascending j, so
// each position's list is in ascending j): at most P positions of the HW get a gradient, and no thread scans all P argmins
// per channel.  Then per position h, threads over channels: dx[n, h, :] = sum over the prototypes j of h's list, in
// ascending j, of g[n, j] (z - p_j) / d[n, j]; times z (1 - z) with `act`.  Every position is written (0 off the argmins).
// With `act`, dx is the operand of the neck's dgrad / wgrad MMAs and `round` stores it rounded to tf32.
__global__ void pt_dist_bwd_x_kernel(const float* __restrict__ z, const float* __restrict__ protos,
                                     const float* __restrict__ mind, const int* __restrict__ argmin,
                                     const float* __restrict__ g, float* __restrict__ dx, int HW, int D, int P, int act,
                                     int round) {
  extern __shared__ int grp[];                 // start[HW + 1], then the prototypes ordered by position
  int* start = grp;
  int* list = grp + HW + 1;
  const int n = blockIdx.x;
  const int* am = argmin + (size_t)n * P;
  if (threadIdx.x == 0) {
    for (int h = 0; h <= HW; ++h) start[h] = 0;
    for (int j = 0; j < P; ++j) ++start[am[j] + 1];
    for (int h = 0; h < HW; ++h) start[h + 1] += start[h];
    for (int j = 0; j < P; ++j) list[start[am[j]]++] = j;          // start[h] ends at the end of h's list
    for (int h = HW; h > 0; --h) start[h] = start[h - 1];
    start[0] = 0;
  }
  __syncthreads();
  for (int h = 0; h < HW; ++h) {
    const float* zr = z + ((size_t)n * HW + h) * D;
    float* out = dx + ((size_t)n * HW + h) * D;
    const int j0 = start[h], j1 = start[h + 1];
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      const float zv = zr[d];
      float acc = 0.f;
      for (int i = j0; i < j1; ++i) {
        const int j = list[i];
        const float w = g[(size_t)n * P + j] / mind[(size_t)n * P + j];
        acc = fmaf(w, zv - protos[(size_t)j * D + d], acc);
      }
      if (act) acc *= zv * (1.f - zv);
      out[d] = round ? tf32_round(acc) : acc;
    }
  }
}

// Block per prototype j, threads over channels: dp[j, :] = -sum_n g[n, j] (z[n, argmin] - p_j) / d[n, j], ascending n.
__global__ void pt_dist_bwd_p_kernel(const float* __restrict__ z, const float* __restrict__ protos,
                                     const float* __restrict__ mind, const int* __restrict__ argmin,
                                     const float* __restrict__ g, float* __restrict__ dp, int N, int HW, int D, int P) {
  const int j = blockIdx.x;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const float pv = protos[(size_t)j * D + d];
    float acc = 0.f;
    for (int n = 0; n < N; ++n) {
      const float w = g[(size_t)n * P + j] / mind[(size_t)n * P + j];
      acc = fmaf(w, z[((size_t)n * HW + argmin[(size_t)n * P + j]) * D + d] - pv, acc);
    }
    dp[(size_t)j * D + d] = -acc;
  }
}

// Block per leaf: sm[l, :] = softmax(theta[l, :] - max) (leaf.py:67).
__global__ void pt_leaf_softmax_kernel(const float* __restrict__ theta, float* __restrict__ sm, int K) {
  __shared__ float red[32];
  const float* th = theta + (size_t)blockIdx.x * K;
  float m, s;
  leaf_softmax_stats(th, K, red, m, s);
  for (int k = threadIdx.x; k < K; k += blockDim.x) sm[(size_t)blockIdx.x * K + k] = expf(th[k] - m) / s;
}

// Block per image n.  Top-down, one depth at a time: ps = exp(-mind[branch rank]), left child (1 - ps) pa, right child
// ps pa (branch.py:45-48), kept in shared memory in heap order and stored to pa[n, pre-order index]; then
// pred[n, k] = sum_l pa[leaf l] sm[l, k] in ascending l.
__global__ void pt_route_fwd_kernel(const float* __restrict__ mind, const float* __restrict__ sm, float* __restrict__ ps,
                                    float* __restrict__ pa, float* __restrict__ pred, int H, int K) {
  extern __shared__ float heap[];
  const int n = blockIdx.x, P = (1 << H) - 1, nodes = 2 * P + 1, L = 1 << H;
  if (threadIdx.x == 0) heap[0] = 1.f;
  __syncthreads();
  for (int d = 0; d < H; ++d) {
    for (int q = threadIdx.x; q < (1 << d); q += blockDim.x) {
      const int r = pt_branch(d, q, H);
      const float p = expf(-mind[(size_t)n * P + r]);
      const float a = heap[(1 << d) - 1 + q];
      ps[(size_t)n * P + r] = p;
      pa[(size_t)n * nodes + pt_node(d, q, H)] = a;
      heap[(2 << d) - 1 + 2 * q] = (1.f - p) * a;
      heap[(2 << d) + 2 * q] = p * a;
    }
    __syncthreads();
  }
  const float* pl = heap + L - 1;
  for (int q = threadIdx.x; q < L; q += blockDim.x) pa[(size_t)n * nodes + pt_node(H, q, H)] = pl[q];
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float acc = 0.f;
    for (int l = 0; l < L; ++l) acc = fmaf(pl[l], sm[(size_t)l * K + k], acc);
    pred[(size_t)n * K + k] = acc;
  }
}

// Block per image n, bottom-up.  u[leaf l] = dpred[n, :] . sm[l, :] (a warp per leaf, lane-strided, fixed xor tree);
// u[branch] = (1 - ps) u[left] + ps u[right], so dL/dps = pa (u[right] - u[left]) and, through ps = exp(-mind),
// dmind = -ps pa (u[right] - u[left]).  No division by ps or 1 - ps.
__global__ void pt_route_bwd_kernel(const float* __restrict__ ps, const float* __restrict__ pa, const float* __restrict__ sm,
                                    const float* __restrict__ dpred, float* __restrict__ dmind, int H, int K) {
  extern __shared__ float heap[];
  const int n = blockIdx.x, P = (1 << H) - 1, nodes = 2 * P + 1, L = 1 << H;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* gr = dpred + (size_t)n * K;
  for (int l = warp; l < L; l += nw) {
    const float* s = sm + (size_t)l * K;
    float u = 0.f;
    for (int k = lane; k < K; k += 32) u = fmaf(gr[k], s[k], u);
    u = warp_sum(u);
    if (lane == 0) heap[L - 1 + l] = u;
  }
  __syncthreads();
  for (int d = H - 1; d >= 0; --d) {
    for (int q = threadIdx.x; q < (1 << d); q += blockDim.x) {
      const int r = pt_branch(d, q, H);
      const float p = ps[(size_t)n * P + r];
      const float ul = heap[(2 << d) - 1 + 2 * q], ur = heap[(2 << d) + 2 * q];
      heap[(1 << d) - 1 + q] = (1.f - p) * ul + p * ur;
      dmind[(size_t)n * P + r] = -p * (pa[(size_t)n * nodes + pt_node(d, q, H)] * (ur - ul));
    }
    __syncthreads();
  }
}

// Block per leaf l: G[k] = sum_n pa[n, leaf l] dpred[n, k] (ascending n), then the softmax adjoint
// dtheta[l, k] = sm[l, k] (G[k] - sum_j G[j] sm[l, j]).
__global__ void pt_dtheta_kernel(const float* __restrict__ pa, const float* __restrict__ sm, const float* __restrict__ dpred,
                                 float* __restrict__ dtheta, int N, int H, int K) {
  extern __shared__ float G[];
  __shared__ float red[32];
  const int l = blockIdx.x, nodes = (2 << H) - 1;
  const int leaf = pt_node(H, l, H);
  const float* s = sm + (size_t)l * K;
  float dot = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float acc = 0.f;
    for (int n = 0; n < N; ++n) acc = fmaf(pa[(size_t)n * nodes + leaf], dpred[(size_t)n * K + k], acc);
    G[k] = acc;
    dot = fmaf(acc, s[k], dot);
  }
  dot = block_sum(dot, red);
  for (int k = threadIdx.x; k < K; k += blockDim.x) dtheta[(size_t)l * K + k] = s[k] * (G[k] - dot);
}

// One block.  V = the rows with a label in [0, K) (F.nll_loss's mean runs over the rows it does not ignore); warp w takes rows
// w, w + 32, ...: loss term -log pred[r, y], dpred[r, :] = -onehot(y) / (V pred[r, y]) and the top-1 hit (first maximum).
// A label outside [0, K) gets no term and never counts.  Per-warp fp64 sums, folded in warp order.
__global__ void pt_nll_kernel(const float* __restrict__ pred, const long long* __restrict__ labels, int R, int K,
                              float* __restrict__ loss, float* __restrict__ dpred, int* __restrict__ correct) {
  __shared__ double s_loss[32];
  __shared__ int s_int[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  int v = 0;
  for (int r = threadIdx.x; r < R; r += blockDim.x) v += labels[r] >= 0 && labels[r] < K;
  const int V = block_sum(v, s_int);
  double acc = 0.0;
  int hits = 0;
  for (int r = warp; r < R; r += nw) {
    const float* z = pred + (size_t)r * K;
    const long long y = labels[r];
    const bool valid = y >= 0 && y < K;
    const float py = valid ? z[y] : 1.f;
    float best = -INFINITY;
    int am = 0;
    for (int k = lane; k < K; k += 32) {
      const float v = z[k];
      if (v > best) { best = v; am = k; }
      dpred[(size_t)r * K + k] = (valid && k == y) ? -1.f / ((float)V * py) : 0.f;
    }
    warp_argmax(best, am);
    if (lane == 0 && valid) {
      acc -= (double)logf(py);
      hits += (am == y);
    }
  }
  const double t = block_sum(acc, s_loss);     // acc, hits are 0 outside lane 0
  const int h = block_sum(hits, s_int);
  if (threadIdx.x == 0) {
    loss[0] = (float)(t / V);                   // no valid row: 0 / 0, NaN, as F.nll_loss gives
    if (correct) correct[0] = h;
  }
}

// Block per leaf l (Examples/ProtoTreeNet.py:116-127): with sm = softmax(theta[l]),
// update[l, k] = sum_b [y_b = k] (pa[b, leaf l] sm[k]) / pred[b, k], in ascending b.
__global__ void pt_leaf_update_sum_kernel(const float* __restrict__ theta, const float* __restrict__ pa,
                                          const float* __restrict__ pred, const long long* __restrict__ labels,
                                          float* __restrict__ update, int N, int H, int K) {
  __shared__ float red[32];
  const int l = blockIdx.x, nodes = (2 << H) - 1;
  const int leaf = pt_node(H, l, H);
  const float* th = theta + (size_t)l * K;
  float m, s;
  leaf_softmax_stats(th, K, red, m, s);
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float smk = expf(th[k] - m) / s;
    float upd = 0.f;
    for (int b = 0; b < N; ++b)
      if (labels[b] == k) upd += (pa[(size_t)b * nodes + leaf] * smk) / pred[(size_t)b * K + k];
    update[(size_t)l * K + k] = upd;
  }
}

// theta = relu(theta - theta0 / num_batches) + update (Examples/ProtoTreeNet.py:128-132), elementwise.
__global__ void pt_leaf_update_apply_kernel(float* __restrict__ theta, const float* __restrict__ theta0,
                                            const float* __restrict__ update, size_t n, float num_batches) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    theta[i] = fmaxf(theta[i] - theta0[i] / num_batches, 0.f) + update[i];
}

static int check_tree(int N, int H, int K, const char* op) {
  HK_REQUIRE(N > 0 && K > 0 && H >= 1, HK_ERR_ARG, "%s: N=%d height=%d K=%d", op, N, H, K);
  HK_REQUIRE(H <= PT_MAX_HEIGHT, HK_ERR_UNSUPPORTED, "%s: height=%d above %d", op, H, PT_MAX_HEIGHT);
  return 0;
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_prototree_dist_fwd(const float* x, const float* protos, float* z, float* mind, int* argmin, int N, int HW, int D,
                          int P, int act, void* stream) {
  HK_REQUIRE(x && protos && mind && argmin && (!act || z), HK_ERR_ARG, "hk_prototree_dist_fwd: null pointer");
  HK_REQUIRE(N > 0 && HW > 0 && D > 0 && P > 0, HK_ERR_ARG, "hk_prototree_dist_fwd: N=%d HW=%d D=%d P=%d", N, HW, D, P);
  HK_REQUIRE(N <= 65535, HK_ERR_UNSUPPORTED, "hk_prototree_dist_fwd: N=%d above 65535", N);
  pt_dist_fwd_kernel<<<dim3((P + PT_TP - 1) / PT_TP, N), 256, 0, (cudaStream_t)stream>>>(x, protos, z, mind, argmin, HW, D,
                                                                                         P, act);
  HK_LAUNCH_CHECK("pt_dist_fwd_kernel");
  return 0;
}

int hk_prototree_dist_bwd(const float* z, const float* protos, const float* mind, const int* argmin, const float* dmind,
                          float* dx, float* dprotos, int N, int HW, int D, int P, int act, void* stream) {
  HK_REQUIRE(z && protos && mind && argmin && dmind && dx && dprotos, HK_ERR_ARG, "hk_prototree_dist_bwd: null pointer");
  HK_REQUIRE(N > 0 && HW > 0 && D > 0 && P > 0, HK_ERR_ARG, "hk_prototree_dist_bwd: N=%d HW=%d D=%d P=%d", N, HW, D, P);
  const size_t grp = (size_t)(HW + 1 + P) * sizeof(int);
  HK_REQUIRE(grp <= PT_MAX_GROUP_BYTES, HK_ERR_UNSUPPORTED, "hk_prototree_dist_bwd: HW + P = %d above %d", HW + P,
             (int)(PT_MAX_GROUP_BYTES / sizeof(int)) - 1);
  if (int r = allow_dynamic_smem<pt_dist_bwd_x_kernel>(PT_MAX_GROUP_BYTES, "pt_dist_bwd_x_kernel")) return r;
  const int tpb = D >= 256 ? 256 : (D + 31) / 32 * 32;
  pt_dist_bwd_x_kernel<<<N, tpb, grp, (cudaStream_t)stream>>>(z, protos, mind, argmin, dmind, dx, HW, D, P, act,
                                                             act && !precise() ? 1 : 0);
  HK_LAUNCH_CHECK("pt_dist_bwd_x_kernel");
  pt_dist_bwd_p_kernel<<<P, tpb, 0, (cudaStream_t)stream>>>(z, protos, mind, argmin, dmind, dprotos, N, HW, D, P);
  HK_LAUNCH_CHECK("pt_dist_bwd_p_kernel");
  return 0;
}

int hk_prototree_route_fwd(const float* mind, const float* theta, float* sm, float* ps, float* pa, float* pred, int N,
                           int height, int K, void* stream) {
  HK_REQUIRE(mind && theta && sm && ps && pa && pred, HK_ERR_ARG, "hk_prototree_route_fwd: null pointer");
  if (int r = check_tree(N, height, K, "hk_prototree_route_fwd")) return r;
  const int L = 1 << height;
  pt_leaf_softmax_kernel<<<L, 256, 0, (cudaStream_t)stream>>>(theta, sm, K);
  HK_LAUNCH_CHECK("pt_leaf_softmax_kernel");
  pt_route_fwd_kernel<<<N, 256, (size_t)(2 * L - 1) * sizeof(float), (cudaStream_t)stream>>>(mind, sm, ps, pa, pred, height,
                                                                                            K);
  HK_LAUNCH_CHECK("pt_route_fwd_kernel");
  return 0;
}

int hk_prototree_route_bwd(const float* ps, const float* pa, const float* sm, const float* dpred, float* dmind,
                           float* dtheta, int N, int height, int K, void* stream) {
  HK_REQUIRE(ps && pa && sm && dpred && dmind, HK_ERR_ARG, "hk_prototree_route_bwd: null pointer");
  if (int r = check_tree(N, height, K, "hk_prototree_route_bwd")) return r;
  HK_REQUIRE(!dtheta || K <= PT_MAX_K, HK_ERR_UNSUPPORTED, "hk_prototree_route_bwd: dtheta needs K <= %d (K=%d)", PT_MAX_K,
             K);
  const int L = 1 << height;
  pt_route_bwd_kernel<<<N, 256, (size_t)(2 * L - 1) * sizeof(float), (cudaStream_t)stream>>>(ps, pa, sm, dpred, dmind,
                                                                                             height, K);
  HK_LAUNCH_CHECK("pt_route_bwd_kernel");
  if (dtheta) {
    if (int r = allow_dynamic_smem<pt_dtheta_kernel>(PT_MAX_K * sizeof(float), "pt_dtheta_kernel")) return r;
    pt_dtheta_kernel<<<L, 256, (size_t)K * sizeof(float), (cudaStream_t)stream>>>(pa, sm, dpred, dtheta, N, height, K);
    HK_LAUNCH_CHECK("pt_dtheta_kernel");
  }
  return 0;
}

int hk_prototree_nll(const float* pred, const long long* labels, float* loss, float* dpred, int* correct, int N, int K,
                     void* stream) {
  HK_REQUIRE(pred && labels && loss && dpred, HK_ERR_ARG, "hk_prototree_nll: null pointer");
  HK_REQUIRE(N > 0 && K > 0, HK_ERR_ARG, "hk_prototree_nll: N=%d K=%d", N, K);
  pt_nll_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(pred, labels, N, K, loss, dpred, correct);
  HK_LAUNCH_CHECK("pt_nll_kernel");
  return 0;
}

int hk_prototree_leaf_update_sum(const float* theta, const float* pa, const float* pred, const long long* labels,
                                 float* update, int N, int height, int K, void* stream) {
  HK_REQUIRE(theta && pa && pred && labels && update, HK_ERR_ARG, "hk_prototree_leaf_update_sum: null pointer");
  if (int r = check_tree(N, height, K, "hk_prototree_leaf_update_sum")) return r;
  pt_leaf_update_sum_kernel<<<1 << height, 256, 0, (cudaStream_t)stream>>>(theta, pa, pred, labels, update, N, height, K);
  HK_LAUNCH_CHECK("pt_leaf_update_sum_kernel");
  return 0;
}

int hk_prototree_leaf_update_apply(float* theta, const float* theta0, const float* update, int height, int K,
                                   float num_batches, void* stream) {
  HK_REQUIRE(theta && theta0 && update, HK_ERR_ARG, "hk_prototree_leaf_update_apply: null pointer");
  if (int r = check_tree(1, height, K, "hk_prototree_leaf_update_apply")) return r;
  HK_REQUIRE(num_batches > 0.f, HK_ERR_ARG, "hk_prototree_leaf_update_apply: num_batches=%g", (double)num_batches);
  const size_t n = ((size_t)1 << height) * K;
  pt_leaf_update_apply_kernel<<<grid_1d(n, 256), 256, 0, (cudaStream_t)stream>>>(theta, theta0, update, n, num_batches);
  HK_LAUNCH_CHECK("pt_leaf_update_apply_kernel");
  return 0;
}

}  // extern "C"
