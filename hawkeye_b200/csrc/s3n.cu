// S3N, selective sparse sampling (reference model/methods/S3N.py): the sampler that turns the class response maps into
// the two 31x31 sampling maps (generate_map, :193-270), the grid each map gives (create_grid, :156-191), the image warp
// (F.interpolate of the grid to the image size + F.grid_sample, :186 and :274-282), their backward passes, and the image
// gradient of the ResNet stem (the 7x7 stride-2 conv, reference backbone/resnet.py:176) that the warp's backward needs.
// Every reduction runs in a fixed order: no atomics, the same bits on every run.
#include "common.cuh"
#include "host.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

constexpr int S3N_G = 31;                       // grid_size
constexpr int S3N_GG = S3N_G * S3N_G;
constexpr int S3N_PAD = 30;                     // padding_size
constexpr int S3N_M = S3N_G + 2 * S3N_PAD;      // global_size: 91
constexpr int S3N_F = 2 * S3N_PAD + 1;          // filter size: 61
constexpr int S3N_FF = S3N_F * S3N_F;
constexpr int S3N_MAX_K = 4096;                 // classes the sampler keeps in shared memory
constexpr int S3N_MAX_HW = 64;                  // side of a class response map (14 at 448)
constexpr int S3N_ZOOM = 1, S3N_INV = 2;        // peak record flags: which map the peak adds to

// align_corners=True source coordinate of output index o, as upsample_bilinear2d computes it: (i0, i1, lambda1)
__device__ __forceinline__ void s3n_src(int o, float scale, int in, int& i0, int& i1, float& l1) {
  const float src = scale * (float)o;
  i0 = (int)src;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = fminf(fmaxf(src - (float)i0, 0.f), 1.f);
}

__device__ __forceinline__ float s3n_scale(int in, int out) { return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f; }

// Block (image n): S3N.py:193-270 on the maps of the raw branch's 1x1 conv, crm [N, h, w, K] (the GEMM's NHWC rows).
//  1. the spatial mean of each class's 31x31 interpolated map, as weights of the h x w map (the interpolation is linear);
//  2. softmax, top-5 and gate_score = sum p log p; the decision map is the top-1 class's interpolated map when the gate
//     exceeds -0.2, else the mean of the top-5 maps; min-max normalised;
//  3. peaks: the first maximum of its 3x3 window (-inf padding) that is >= the map's mean, in row-major order;
//  4. the assignment by p (0: both maps; 1: the zoom map when s > u at the peak's position, else the complementary one;
//     2: the first maximum-score peak to the zoom map, the first minimum-score peak to the complementary one);
//  5. xs[n] = base + sum s G(radius sqrt s), xs[N + n] = base + sum (1/s) G(radius_inv sqrt s), G(t) = exp(-d^2/2(31t)^2).
// A map without peaks (a constant map normalises to NaN) leaves both maps at base.
__global__ void __launch_bounds__(1024) s3n_sample_maps_kernel(
    const float* __restrict__ crm, const float* __restrict__ rnd, const int* __restrict__ pp,
    const float* __restrict__ radius, const float* __restrict__ radius_inv, float base, float* __restrict__ xs,
    int* __restrict__ peaks, float* __restrict__ scores, int* __restrict__ counts, int N, int h, int w, int K) {
  __shared__ float mean_k[S3N_MAX_K];
  __shared__ float wy[S3N_MAX_HW], wx[S3N_MAX_HW];
  __shared__ float dm[S3N_GG];
  __shared__ float red[32];
  __shared__ int redi[32];
  __shared__ int top[5];
  __shared__ float topp[5];
  __shared__ int use_top1;
  __shared__ int pos_s[S3N_GG];
  __shared__ int flag_s[S3N_GG];
  __shared__ int warp_off[33];
  const int n = blockIdx.x, t = threadIdx.x, nt = blockDim.x;
  const float* m = crm + (size_t)n * h * w * K;
  const float sy = s3n_scale(h, S3N_G), sx = s3n_scale(w, S3N_G);

  // 1. column / row weights of the interpolation: mean over the 31x31 map = sum_yx wy[y] wx[x] crm[y, x] / 961
  if (t < h || (t >= S3N_MAX_HW && t - S3N_MAX_HW < w)) {
    const bool isy = t < h;
    const int i = isy ? t : t - S3N_MAX_HW, in = isy ? h : w;
    const float sc = isy ? sy : sx;
    float acc = 0.f;
    for (int o = 0; o < S3N_G; ++o) {
      int i0, i1;
      float l1;
      s3n_src(o, sc, in, i0, i1, l1);
      if (i0 == i) acc += 1.f - l1;
      if (i1 == i) acc += l1;
    }
    (isy ? wy : wx)[i] = acc;
  }
  __syncthreads();
  float lmax = -INFINITY;
  for (int k = t; k < K; k += nt) {
    float acc = 0.f;
    for (int y = 0; y < h; ++y) {
      float r = 0.f;
      for (int x = 0; x < w; ++x) r = fmaf(wx[x], m[((size_t)y * w + x) * K + k], r);
      acc = fmaf(wy[y], r, acc);
    }
    mean_k[k] = acc / (float)S3N_GG;
    lmax = fmaxf(lmax, mean_k[k]);
  }
  // 2. softmax over the classes, top-5, gate
  const float mx = block_max(lmax, red);
  float se = 0.f;
  for (int k = t; k < K; k += nt) se += expf(mean_k[k] - mx);
  se = block_sum(se, red);
  for (int r = 0; r < 5; ++r) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int k = t; k < K; k += nt) {
      bool taken = false;
      for (int q = 0; q < r; ++q) taken |= top[q] == k;
      if (!taken && mean_k[k] > best) { best = mean_k[k]; bi = k; }
    }
    warp_argmax(best, bi);
    __syncthreads();
    if ((t & 31) == 0) { red[t >> 5] = best; redi[t >> 5] = bi; }
    __syncthreads();
    if (t == 0) {
      float b = red[0];
      int bk = redi[0];
      for (int i = 1; i < nt / 32; ++i)
        if (red[i] > b || (red[i] == b && redi[i] < bk)) { b = red[i]; bk = redi[i]; }
      top[r] = bk;
      topp[r] = expf(b - mx) / se;
    }
    __syncthreads();
  }
  if (t == 0) {
    float g = 0.f;
    for (int r = 0; r < 5; ++r) g += topp[r] * logf(topp[r]);
    use_top1 = g > -0.2f;
  }
  __syncthreads();
  // the decision map, interpolated to 31x31
  float v = 0.f;
  if (t < S3N_GG) {
    int y0, y1, x0, x1;
    float ly, lx;
    s3n_src(t / S3N_G, sy, h, y0, y1, ly);
    s3n_src(t % S3N_G, sx, w, x0, x1, lx);
    const int nc = use_top1 ? 1 : 5;
    for (int r = 0; r < nc; ++r) {
      const int k = top[r];
      const float a00 = m[((size_t)y0 * w + x0) * K + k], a01 = m[((size_t)y0 * w + x1) * K + k];
      const float a10 = m[((size_t)y1 * w + x0) * K + k], a11 = m[((size_t)y1 * w + x1) * K + k];
      v += (1.f - ly) * ((1.f - lx) * a00 + lx * a01) + ly * ((1.f - lx) * a10 + lx * a11);
    }
    if (!use_top1) v = v / 5.f;
  }
  const float vmax = block_max(t < S3N_GG ? v : -INFINITY, red);
  const float vmin = -block_max(t < S3N_GG ? -v : -INFINITY, red);
  const bool flat = !(vmax > vmin);
  if (t < S3N_GG) {
    v = (v - vmin) / (vmax - vmin);
    dm[t] = v;
  }
  const float vmean = block_sum(t < S3N_GG ? v : 0.f, red) / (float)S3N_GG;
  // 3. peaks
  bool peak = false;
  if (t < S3N_GG && !flat) {
    const int y = t / S3N_G, x = t % S3N_G;
    peak = v >= vmean;
    for (int dy = -1; dy <= 1 && peak; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int yy = y + dy, xx = x + dx;
        if ((dy == 0 && dx == 0) || yy < 0 || yy >= S3N_G || xx < 0 || xx >= S3N_G) continue;
        const float u = dm[yy * S3N_G + xx];
        const bool before = dy < 0 || (dy == 0 && dx < 0);        // earlier in the window's row-major order
        if (before ? !(u < v) : !(u <= v)) { peak = false; break; }
      }
  }
  const unsigned bal = __ballot_sync(0xffffffffu, peak);
  if ((t & 31) == 0) warp_off[t >> 5] = __popc(bal);
  __syncthreads();
  if (t == 0) {
    int acc = 0;
    for (int i = 0; i < nt / 32; ++i) { const int c = warp_off[i]; warp_off[i] = acc; acc += c; }
    warp_off[32] = acc;
  }
  __syncthreads();
  const int np = warp_off[32];
  if (peak) pos_s[warp_off[t >> 5] + __popc(bal & ((1u << (t & 31)) - 1u))] = t;
  __syncthreads();
  // 4. assignment
  const int p = pp[0];
  if (p == 2) {
    if (t == 0) {
      int imax = 0, imin = 0;
      for (int i = 0; i < np; ++i) {
        flag_s[i] = 0;
        if (dm[pos_s[i]] > dm[pos_s[imax]]) imax = i;
        if (dm[pos_s[i]] < dm[pos_s[imin]]) imin = i;
      }
      if (np > 0) { flag_s[imax] |= S3N_ZOOM; flag_s[imin] |= S3N_INV; }
    }
  } else {
    for (int i = t; i < np; i += nt) {
      const float s = dm[pos_s[i]];
      flag_s[i] = p == 0 ? (S3N_ZOOM | S3N_INV) : (s > rnd[(size_t)n * S3N_GG + pos_s[i]] ? S3N_ZOOM : S3N_INV);
    }
  }
  __syncthreads();
  for (int i = t; i < np; i += nt) {
    peaks[(size_t)n * S3N_GG + i] = pos_s[i] | (flag_s[i] << 16);
    scores[(size_t)n * S3N_GG + i] = dm[pos_s[i]];
  }
  if (t == 0) counts[n] = np;
  // 5. the two maps
  if (t < S3N_GG) {
    const float r = radius[0], ri = radius_inv[0];
    const int y = t / S3N_G, x = t % S3N_G;
    float z = base, c = base;
    for (int i = 0; i < np; ++i) {
      const int q = pos_s[i];
      const float s = dm[q];
      const float dy = (float)(y - q / S3N_G), dx = (float)(x - q % S3N_G);
      const float d2 = dx * dx + dy * dy;
      if (flag_s[i] & S3N_ZOOM) {
        const float th = sqrtf(s) * r * (float)S3N_G;
        z += s * expf(-0.5f * d2 / (th * th));
      }
      if (flag_s[i] & S3N_INV) {
        const float th = sqrtf(s) * ri * (float)S3N_G;
        c += (1.f / s) * expf(-0.5f * d2 / (th * th));
      }
    }
    xs[(size_t)n * S3N_GG + t] = z;
    xs[((size_t)N + n) * S3N_GG + t] = c;
  }
}

// One block: dradius = sum over images, peaks of the zoom map and positions of dxs s dG/dr, dradius_inv likewise over the
// complementary map; each thread owns positions, then the fixed-order block sum.
__global__ void __launch_bounds__(1024) s3n_sample_maps_bwd_kernel(
    const float* __restrict__ dxs, const int* __restrict__ peaks, const float* __restrict__ scores,
    const int* __restrict__ counts, const float* __restrict__ radius, const float* __restrict__ radius_inv,
    float* __restrict__ dradius, float* __restrict__ dradius_inv, int N) {
  __shared__ float red[32];
  const int t = threadIdx.x;
  const float r = radius[0], ri = radius_inv[0];
  float ar = 0.f, ai = 0.f;
  if (t < S3N_GG) {
    const int y = t / S3N_G, x = t % S3N_G;
    for (int n = 0; n < N; ++n) {
      const float gz = dxs[(size_t)n * S3N_GG + t], gc = dxs[((size_t)N + n) * S3N_GG + t];
      for (int i = 0; i < counts[n]; ++i) {
        const int rec = peaks[(size_t)n * S3N_GG + i], q = rec & 0xffff, f = rec >> 16;
        const float s = scores[(size_t)n * S3N_GG + i];
        const float dy = (float)(y - q / S3N_G), dx = (float)(x - q % S3N_G);
        const float d2 = dx * dx + dy * dy;
        // d/dr [c exp(-d2 / 2 th^2)], th = 31 r sqrt(s): c exp(...) d2 / (th^2 r)
        if (f & S3N_ZOOM) {
          const float th = sqrtf(s) * r * (float)S3N_G, th2 = th * th;
          ar = fmaf(gz, s * expf(-0.5f * d2 / th2) * d2 / (th2 * r), ar);
        }
        if (f & S3N_INV) {
          const float th = sqrtf(s) * ri * (float)S3N_G, th2 = th * th;
          ai = fmaf(gc, (1.f / s) * expf(-0.5f * d2 / th2) * d2 / (th2 * ri), ai);
        }
      }
    }
  }
  ar = block_sum(ar, red);
  ai = block_sum(ai, red);
  if (t == 0) { dradius[0] = ar; dradius_inv[0] = ai; }
}

// replication-padded map value at padded position (u, v)
__device__ __forceinline__ float s3n_padded(const float* mp, int u, int v) {
  const int r = min(max(u - S3N_PAD, 0), S3N_G - 1), c = min(max(v - S3N_PAD, 0), S3N_G - 1);
  return mp[r * S3N_G + c];
}

__device__ __forceinline__ float s3n_basis(int i) { return (float)(i - S3N_PAD) / (float)(S3N_G - 1); }

// Block (image b), thread (i, j) of the 31x31 grid: S0, Sx, Sy = the 61x61 correlations of the padded map, of the map times
// the x basis (column) and of the map times the y basis (row); grid = clamp(2 S / S0 - 1, -1, 1).
__global__ void __launch_bounds__(S3N_G * 32) s3n_grid_fwd_kernel(const float* __restrict__ maps,
                                                                  const float* __restrict__ filt, float* __restrict__ grid,
                                                                  float* __restrict__ sums) {
  __shared__ float mp[S3N_M * S3N_M];
  __shared__ float fs[S3N_FF];
  const int b = blockIdx.x, t = threadIdx.x;
  const float* src = maps + (size_t)b * S3N_GG;
  for (int k = t; k < S3N_M * S3N_M; k += blockDim.x) mp[k] = s3n_padded(src, k / S3N_M, k % S3N_M);
  for (int k = t; k < S3N_FF; k += blockDim.x) fs[k] = filt[k];
  __syncthreads();
  const int i = t >> 5, j = t & 31;
  if (j >= S3N_G) return;
  float s0 = 0.f, sxx = 0.f, syy = 0.f;
  for (int a = 0; a < S3N_F; ++a) {
    const float py = s3n_basis(i + a);
    const float* row = mp + (i + a) * S3N_M + j;
    const float* fr = fs + a * S3N_F;
    for (int c = 0; c < S3N_F; ++c) {
      const float f = fr[c], m = row[c];
      s0 = fmaf(f, m, s0);
      sxx = fmaf(f, m * s3n_basis(j + c), sxx);
      syy = fmaf(f, m * py, syy);
    }
  }
  const size_t o = (size_t)b * S3N_GG + i * S3N_G + j;
  grid[o * 2] = fminf(fmaxf(sxx / s0 * 2.f - 1.f, -1.f), 1.f);
  grid[o * 2 + 1] = fminf(fmaxf(syy / s0 * 2.f - 1.f, -1.f), 1.f);
  sums[o * 3] = s0;
  sums[o * 3 + 1] = sxx;
  sums[o * 3 + 2] = syy;
}

// The gradients at S0, Sx, Sy of grid position o from dgrid: the clamp passes where -1 <= 2 S / S0 - 1 <= 1 (inclusive,
// as torch.clamp), then the quotient rule.
__device__ __forceinline__ void s3n_dsums(const float* sums, const float* dgrid, size_t o, float& g0, float& gx, float& gy) {
  const float s0 = sums[o * 3], sxx = sums[o * 3 + 1], syy = sums[o * 3 + 2];
  const float vx = sxx / s0 * 2.f - 1.f, vy = syy / s0 * 2.f - 1.f;
  const float dx = (vx >= -1.f && vx <= 1.f) ? dgrid[o * 2] : 0.f;
  const float dy = (vy >= -1.f && vy <= 1.f) ? dgrid[o * 2 + 1] : 0.f;
  gx = 2.f * dx / s0;
  gy = 2.f * dy / s0;
  g0 = -(gx * sxx + gy * syy) / s0;
}

// Block (padded row u, image b), thread v: the gradient at the padded map, dMp[u, v] = A0 + px(v) Ax + py(u) Ay with
// A = sum over grid positions (i, j) of filter[u - i, v - j] times (g0, gx, gy)[i, j].
__global__ void __launch_bounds__(128) s3n_grid_bwd_pad_kernel(const float* __restrict__ filt,
                                                               const float* __restrict__ sums,
                                                               const float* __restrict__ dgrid, float* __restrict__ dmp) {
  __shared__ float fs[S3N_FF];
  __shared__ float gs[3][S3N_GG];
  const int u = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  for (int k = t; k < S3N_FF; k += blockDim.x) fs[k] = filt[k];
  for (int k = t; k < S3N_GG; k += blockDim.x) s3n_dsums(sums, dgrid, (size_t)b * S3N_GG + k, gs[0][k], gs[1][k], gs[2][k]);
  __syncthreads();
  if (t >= S3N_M) return;
  const int v = t;
  float a0 = 0.f, ax = 0.f, ay = 0.f;
  const int i0 = max(0, u - (S3N_F - 1)), i1 = min(S3N_G - 1, u);
  const int j0 = max(0, v - (S3N_F - 1)), j1 = min(S3N_G - 1, v);
  for (int i = i0; i <= i1; ++i)
    for (int j = j0; j <= j1; ++j) {
      const float f = fs[(u - i) * S3N_F + (v - j)];
      const int k = i * S3N_G + j;
      a0 = fmaf(f, gs[0][k], a0);
      ax = fmaf(f, gs[1][k], ax);
      ay = fmaf(f, gs[2][k], ay);
    }
  dmp[((size_t)b * S3N_M + u) * S3N_M + v] = a0 + s3n_basis(v) * ax + s3n_basis(u) * ay;
}

// The adjoint of the replication pad: dmaps[b, r, c] = sum of dMp over the padded positions that copy (r, c), row-major.
__global__ void s3n_grid_bwd_fold_kernel(const float* __restrict__ dmp, float* __restrict__ dmaps, int B) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < B * S3N_GG; k += gridDim.x * blockDim.x) {
    const int b = k / S3N_GG, r = (k % S3N_GG) / S3N_G, c = k % S3N_G;
    const int u0 = r == 0 ? 0 : r + S3N_PAD, u1 = r == S3N_G - 1 ? S3N_M - 1 : r + S3N_PAD;
    const int v0 = c == 0 ? 0 : c + S3N_PAD, v1 = c == S3N_G - 1 ? S3N_M - 1 : c + S3N_PAD;
    const float* d = dmp + (size_t)b * S3N_M * S3N_M;
    float acc = 0.f;
    for (int u = u0; u <= u1; ++u)
      for (int v = v0; v <= v1; ++v) acc += d[u * S3N_M + v];
    dmaps[k] = acc;
  }
}

// Block (filter row a, image b), thread c: image b's share of dfilter[a, c] = sum over grid positions (i, j) of
// Mp[i + a, j + c] (g0 + gx px(j + c) + gy py(i + a))[i, j].
__global__ void __launch_bounds__(64) s3n_grid_bwd_filter_kernel(const float* __restrict__ maps,
                                                                 const float* __restrict__ sums,
                                                                 const float* __restrict__ dgrid,
                                                                 float* __restrict__ part) {
  __shared__ float rows[S3N_G * S3N_M];
  __shared__ float gs[3][S3N_GG];
  const int a = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const float* src = maps + (size_t)b * S3N_GG;
  for (int k = t; k < S3N_G * S3N_M; k += blockDim.x) rows[k] = s3n_padded(src, a + k / S3N_M, k % S3N_M);
  for (int k = t; k < S3N_GG; k += blockDim.x) s3n_dsums(sums, dgrid, (size_t)b * S3N_GG + k, gs[0][k], gs[1][k], gs[2][k]);
  __syncthreads();
  if (t >= S3N_F) return;
  const int c = t;
  float acc = 0.f;
  for (int i = 0; i < S3N_G; ++i) {
    const float py = s3n_basis(i + a);
    for (int j = 0; j < S3N_G; ++j) {
      const int k = i * S3N_G + j;
      const float g = gs[0][k] + gs[1][k] * s3n_basis(j + c) + gs[2][k] * py;
      acc = fmaf(rows[i * S3N_M + j + c], g, acc);
    }
  }
  part[((size_t)b * S3N_F + a) * S3N_F + c] = acc;
}

__global__ void s3n_grid_bwd_filter_sum_kernel(const float* __restrict__ part, float* __restrict__ dfilt, int B) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < S3N_FF; k += gridDim.x * blockDim.x) {
      float acc = 0.f;
      for (int b = 0; b < B; ++b) acc += part[(size_t)b * S3N_FF + k];
      dfilt[k] = acc;
  }
}

// The coarse grid upsampled (align_corners=True) to output pixel (oy, ox) of a Ho x Wo image -> (gx, gy)
__device__ __forceinline__ void s3n_fine_grid(const float* g, int oy, int ox, float scy, float scx, float& gx, float& gy) {
  int y0, y1, x0, x1;
  float ly, lx;
  s3n_src(oy, scy, S3N_G, y0, y1, ly);
  s3n_src(ox, scx, S3N_G, x0, x1, lx);
  const float* a00 = g + (y0 * S3N_G + x0) * 2;
  const float* a01 = g + (y0 * S3N_G + x1) * 2;
  const float* a10 = g + (y1 * S3N_G + x0) * 2;
  const float* a11 = g + (y1 * S3N_G + x1) * 2;
  gx = (1.f - ly) * ((1.f - lx) * a00[0] + lx * a01[0]) + ly * ((1.f - lx) * a10[0] + lx * a11[0]);
  gy = (1.f - ly) * ((1.f - lx) * a00[1] + lx * a01[1]) + ly * ((1.f - lx) * a10[1] + lx * a11[1]);
}

// Thread per output pixel of image b: grid_sample(x[b % N], bilinear, zeros, align_corners=True) at the upsampled grid.
__global__ void s3n_warp_fwd_kernel(const float* __restrict__ x, const float* __restrict__ grid, float* __restrict__ out,
                                    int N, int B, int C, int H, int W, int Ho, int Wo) {
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < (size_t)B * Ho * Wo;
       k += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(k / ((size_t)Ho * Wo)), oy = (int)(k / Wo % Ho), ox = (int)(k % Wo);
    float gx, gy;
    s3n_fine_grid(grid + (size_t)b * S3N_GG * 2, oy, ox, s3n_scale(S3N_G, Ho), s3n_scale(S3N_G, Wo), gx, gy);
    const float ix = (gx + 1.f) / 2.f * (float)(W - 1), iy = (gy + 1.f) / 2.f * (float)(H - 1);
    const int xw = (int)floorf(ix), yn = (int)floorf(iy), xe = xw + 1, ys = yn + 1;
    const float wnw = ((float)xe - ix) * ((float)ys - iy), wne = (ix - (float)xw) * ((float)ys - iy);
    const float wsw = ((float)xe - ix) * (iy - (float)yn), wse = (ix - (float)xw) * (iy - (float)yn);
    const bool inw = xw >= 0 && xw < W, ine = xe >= 0 && xe < W, inn = yn >= 0 && yn < H, ins = ys >= 0 && ys < H;
    const float* img = x + (size_t)(b % N) * C * H * W;
    float* o = out + (size_t)b * C * Ho * Wo + (size_t)oy * Wo + ox;
    for (int c = 0; c < C; ++c, img += (size_t)H * W, o += (size_t)Ho * Wo) {
      float v = 0.f;
      if (inn && inw) v += img[yn * W + xw] * wnw;
      if (inn && ine) v += img[yn * W + xe] * wne;
      if (ins && inw) v += img[ys * W + xw] * wsw;
      if (ins && ine) v += img[ys * W + xe] * wse;
      *o = v;
    }
  }
}

// Thread per output pixel: the gradient at the upsampled grid, fine[b, oy, ox, 2] (grid_sampler_2d_backward's grid part).
__global__ void s3n_warp_bwd_fine_kernel(const float* __restrict__ x, const float* __restrict__ grid,
                                         const float* __restrict__ dout, float* __restrict__ fine, int N, int B, int C,
                                         int H, int W, int Ho, int Wo) {
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < (size_t)B * Ho * Wo;
       k += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(k / ((size_t)Ho * Wo)), oy = (int)(k / Wo % Ho), ox = (int)(k % Wo);
    float gx, gy;
    s3n_fine_grid(grid + (size_t)b * S3N_GG * 2, oy, ox, s3n_scale(S3N_G, Ho), s3n_scale(S3N_G, Wo), gx, gy);
    const float ix = (gx + 1.f) / 2.f * (float)(W - 1), iy = (gy + 1.f) / 2.f * (float)(H - 1);
    const int xw = (int)floorf(ix), yn = (int)floorf(iy), xe = xw + 1, ys = yn + 1;
    const bool inw = xw >= 0 && xw < W, ine = xe >= 0 && xe < W, inn = yn >= 0 && yn < H, ins = ys >= 0 && ys < H;
    const float* img = x + (size_t)(b % N) * C * H * W;
    const float* g = dout + (size_t)b * C * Ho * Wo + (size_t)oy * Wo + ox;
    float gix = 0.f, giy = 0.f;
    for (int c = 0; c < C; ++c, img += (size_t)H * W, g += (size_t)Ho * Wo) {
      const float go = *g;
      if (inn && inw) {
        const float v = img[yn * W + xw];
        gix -= v * ((float)ys - iy) * go;
        giy -= v * ((float)xe - ix) * go;
      }
      if (inn && ine) {
        const float v = img[yn * W + xe];
        gix += v * ((float)ys - iy) * go;
        giy -= v * (ix - (float)xw) * go;
      }
      if (ins && inw) {
        const float v = img[ys * W + xw];
        gix -= v * (iy - (float)yn) * go;
        giy += v * ((float)xe - ix) * go;
      }
      if (ins && ine) {
        const float v = img[ys * W + xe];
        gix += v * (iy - (float)yn) * go;
        giy += v * (ix - (float)xw) * go;
      }
    }
    fine[k * 2] = gix * (float)(W - 1) / 2.f;
    fine[k * 2 + 1] = giy * (float)(H - 1) / 2.f;
  }
}

// weight of coarse node ci in the align_corners=True interpolation at output index o
__device__ __forceinline__ float s3n_node_weight(int o, float sc, int ci) {
  int i0, i1;
  float l1;
  s3n_src(o, sc, S3N_G, i0, i1, l1);
  return (i0 == ci ? 1.f - l1 : 0.f) + (i1 == ci ? l1 : 0.f);
}

// Thread per coarse node (b, ci, cj): the adjoint of the upsample, gathered over the output pixels whose interpolation
// reads the node, rows then columns in ascending order.
__global__ void s3n_warp_bwd_coarse_kernel(const float* __restrict__ fine, float* __restrict__ dgrid, int B, int Ho,
                                           int Wo) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < B * S3N_GG; k += gridDim.x * blockDim.x) {
    const int b = k / S3N_GG, ci = (k % S3N_GG) / S3N_G, cj = k % S3N_G;
    const float scy = s3n_scale(S3N_G, Ho), scx = s3n_scale(S3N_G, Wo);
    // the output rows that read node ci have floor(o * scale) in {ci - 1, ci}
    const int oy0 = max(0, (int)((float)(ci - 1) / scy) - 1), oy1 = min(Ho - 1, (int)((float)(ci + 1) / scy) + 1);
    const int ox0 = max(0, (int)((float)(cj - 1) / scx) - 1), ox1 = min(Wo - 1, (int)((float)(cj + 1) / scx) + 1);
    const float* f = fine + (size_t)b * Ho * Wo * 2;
    float ax = 0.f, ay = 0.f;
    for (int oy = oy0; oy <= oy1; ++oy) {
      const float wy = s3n_node_weight(oy, scy, ci);
      if (wy == 0.f) continue;
      float rx = 0.f, ry = 0.f;
      for (int ox = ox0; ox <= ox1; ++ox) {
        const float wx = s3n_node_weight(ox, scx, cj);
        if (wx == 0.f) continue;
        rx = fmaf(wx, f[((size_t)oy * Wo + ox) * 2], rx);
        ry = fmaf(wx, f[((size_t)oy * Wo + ox) * 2 + 1], ry);
      }
      ax = fmaf(wy, rx, ax);
      ay = fmaf(wy, ry, ay);
    }
    dgrid[(size_t)k * 2] = ax;
    dgrid[(size_t)k * 2 + 1] = ay;
  }
}

// Thread per input pixel (n, y, x): dx[n, :, y, x] = sum over the 7x7 taps whose stride-2 output lands on the map and the 64
// output channels of dc[n, oy, ox, o] w[o, :, ky, kx].  The weights sit in shared memory as [ky][kx][o][3].
constexpr int STEM_COUT = 64;
__global__ void __launch_bounds__(256) stem_dgrad_kernel(const float* __restrict__ dc, const float* __restrict__ w,
                                                         float* __restrict__ dx, int N, int H, int W, int Ho, int Wo) {
  __shared__ float ws[49 * STEM_COUT * 3];
  for (int k = threadIdx.x; k < 49 * STEM_COUT * 3; k += blockDim.x) {
    const int c = k % 3, o = k / 3 % STEM_COUT, tap = k / (3 * STEM_COUT);
    ws[k] = w[(o * 3 + c) * 49 + tap];
  }
  __syncthreads();
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < (size_t)N * H * W;
       k += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(k / ((size_t)H * W)), y = (int)(k / W % H), x = (int)(k % W);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int ky = (y + 3) & 1; ky < 7; ky += 2) {
      const int oy = (y + 3 - ky) >> 1;
      if (oy < 0 || oy >= Ho) continue;
      for (int kx = (x + 3) & 1; kx < 7; kx += 2) {
        const int ox = (x + 3 - kx) >> 1;
        if (ox < 0 || ox >= Wo) continue;
        const float4* g = reinterpret_cast<const float4*>(dc + (((size_t)n * Ho + oy) * Wo + ox) * STEM_COUT);
        const float* wt = ws + (ky * 7 + kx) * STEM_COUT * 3;
  #pragma unroll 4
        for (int o4 = 0; o4 < STEM_COUT / 4; ++o4) {
          const float4 gv = g[o4];
          const float gg[4] = {gv.x, gv.y, gv.z, gv.w};
  #pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float* wo = wt + (o4 * 4 + q) * 3;
            a0 = fmaf(gg[q], wo[0], a0);
            a1 = fmaf(gg[q], wo[1], a1);
            a2 = fmaf(gg[q], wo[2], a2);
          }
        }
      }
    }
    const size_t plane = (size_t)H * W, base = (size_t)n * 3 * plane + (size_t)y * W + x;
    dx[base] = a0;
    dx[base + plane] = a1;
    dx[base + 2 * plane] = a2;
  }
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_s3n_sample_maps(const float* crm, const float* rnd, const int* p, const float* radius, const float* radius_inv,
                       float base_ratio, float* xs, int* peaks, float* scores, int* counts, int N, int h, int w, int K,
                       void* stream) {
  HK_REQUIRE(crm && rnd && p && radius && radius_inv && xs && peaks && scores && counts, HK_ERR_ARG,
             "hk_s3n_sample_maps: null pointer");
  HK_REQUIRE(N > 0 && N <= 65535 && h > 0 && w > 0 && K >= 5, HK_ERR_ARG, "hk_s3n_sample_maps: N=%d h=%d w=%d K=%d", N, h,
             w, K);
  HK_REQUIRE(h <= S3N_MAX_HW && w <= S3N_MAX_HW && K <= S3N_MAX_K, HK_ERR_UNSUPPORTED,
             "hk_s3n_sample_maps: maps of %dx%d with %d classes (at most %dx%d and %d classes)", h, w, K, S3N_MAX_HW,
             S3N_MAX_HW, S3N_MAX_K);
  s3n_sample_maps_kernel<<<N, 1024, 0, (cudaStream_t)stream>>>(crm, rnd, p, radius, radius_inv, base_ratio, xs, peaks,
                                                               scores, counts, N, h, w, K);
  HK_LAUNCH_CHECK("s3n_sample_maps_kernel");
  return 0;
}

int hk_s3n_sample_maps_bwd(const float* dxs, const int* peaks, const float* scores, const int* counts,
                           const float* radius, const float* radius_inv, float* dradius, float* dradius_inv, int N,
                           void* stream) {
  HK_REQUIRE(dxs && peaks && scores && counts && radius && radius_inv && dradius && dradius_inv, HK_ERR_ARG,
             "hk_s3n_sample_maps_bwd: null pointer");
  HK_REQUIRE(N > 0, HK_ERR_ARG, "hk_s3n_sample_maps_bwd: N=%d", N);
  s3n_sample_maps_bwd_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(dxs, peaks, scores, counts, radius, radius_inv, dradius,
                                                                   dradius_inv, N);
  HK_LAUNCH_CHECK("s3n_sample_maps_bwd_kernel");
  return 0;
}

int hk_s3n_grid_fwd(const float* maps, const float* filter, float* grid, float* sums, int B, void* stream) {
  HK_REQUIRE(maps && filter && grid && sums, HK_ERR_ARG, "hk_s3n_grid_fwd: null pointer");
  HK_REQUIRE(B > 0, HK_ERR_ARG, "hk_s3n_grid_fwd: B=%d", B);
  s3n_grid_fwd_kernel<<<B, S3N_G * 32, 0, (cudaStream_t)stream>>>(maps, filter, grid, sums);
  HK_LAUNCH_CHECK("s3n_grid_fwd_kernel");
  return 0;
}

size_t hk_s3n_grid_bwd_workspace_bytes(int B) {
  if (B <= 0) return 0;
  const size_t pad = (size_t)B * S3N_M * S3N_M, part = (size_t)B * S3N_FF;
  return (pad + part) * sizeof(float);
}

int hk_s3n_grid_bwd(const float* maps, const float* filter, const float* sums, const float* dgrid, float* dmaps,
                    float* dfilter, int B, void* workspace, size_t workspace_bytes, void* stream) {
  HK_REQUIRE(maps && filter && sums && dgrid && dmaps && dfilter && workspace, HK_ERR_ARG, "hk_s3n_grid_bwd: null pointer");
  HK_REQUIRE(B > 0, HK_ERR_ARG, "hk_s3n_grid_bwd: B=%d", B);
  HK_REQUIRE(workspace_bytes >= hk_s3n_grid_bwd_workspace_bytes(B), HK_ERR_WORKSPACE,
             "hk_s3n_grid_bwd: workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  float* dmp = static_cast<float*>(workspace);
  float* part = dmp + (size_t)B * S3N_M * S3N_M;
  s3n_grid_bwd_pad_kernel<<<dim3(S3N_M, B), 128, 0, s>>>(filter, sums, dgrid, dmp);
  HK_LAUNCH_CHECK("s3n_grid_bwd_pad_kernel");
  s3n_grid_bwd_fold_kernel<<<grid_1d((size_t)B * S3N_GG, 256), 256, 0, s>>>(dmp, dmaps, B);
  HK_LAUNCH_CHECK("s3n_grid_bwd_fold_kernel");
  s3n_grid_bwd_filter_kernel<<<dim3(S3N_F, B), 64, 0, s>>>(maps, sums, dgrid, part);
  HK_LAUNCH_CHECK("s3n_grid_bwd_filter_kernel");
  s3n_grid_bwd_filter_sum_kernel<<<grid_1d(S3N_FF, 256), 256, 0, s>>>(part, dfilter, B);
  HK_LAUNCH_CHECK("s3n_grid_bwd_filter_sum_kernel");
  return 0;
}

int hk_s3n_warp_fwd(const float* x, const float* grid, float* out, int N, int B, int C, int H, int W, int Ho, int Wo,
                    void* stream) {
  HK_REQUIRE(x && grid && out, HK_ERR_ARG, "hk_s3n_warp_fwd: null pointer");
  HK_REQUIRE(N > 0 && B > 0 && B % N == 0 && C > 0 && H > 1 && W > 1 && Ho > 1 && Wo > 1, HK_ERR_ARG,
             "hk_s3n_warp_fwd: N=%d B=%d C=%d H=%d W=%d Ho=%d Wo=%d", N, B, C, H, W, Ho, Wo);
  s3n_warp_fwd_kernel<<<grid_1d((size_t)B * Ho * Wo, 256), 256, 0, (cudaStream_t)stream>>>(x, grid, out, N, B, C, H, W, Ho,
                                                                                            Wo);
  HK_LAUNCH_CHECK("s3n_warp_fwd_kernel");
  return 0;
}

size_t hk_s3n_warp_bwd_workspace_bytes(int B, int Ho, int Wo) {
  if (B <= 0 || Ho <= 0 || Wo <= 0) return 0;
  return (size_t)B * Ho * Wo * 2 * sizeof(float);
}

int hk_s3n_warp_bwd(const float* x, const float* grid, const float* dout, float* dgrid, int N, int B, int C, int H, int W,
                    int Ho, int Wo, void* workspace, size_t workspace_bytes, void* stream) {
  HK_REQUIRE(x && grid && dout && dgrid && workspace, HK_ERR_ARG, "hk_s3n_warp_bwd: null pointer");
  HK_REQUIRE(N > 0 && B > 0 && B % N == 0 && C > 0 && H > 1 && W > 1 && Ho > 1 && Wo > 1, HK_ERR_ARG,
             "hk_s3n_warp_bwd: N=%d B=%d C=%d H=%d W=%d Ho=%d Wo=%d", N, B, C, H, W, Ho, Wo);
  HK_REQUIRE(workspace_bytes >= hk_s3n_warp_bwd_workspace_bytes(B, Ho, Wo), HK_ERR_WORKSPACE,
             "hk_s3n_warp_bwd: workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  float* fine = static_cast<float*>(workspace);
  s3n_warp_bwd_fine_kernel<<<grid_1d((size_t)B * Ho * Wo, 256), 256, 0, s>>>(x, grid, dout, fine, N, B, C, H, W, Ho, Wo);
  HK_LAUNCH_CHECK("s3n_warp_bwd_fine_kernel");
  s3n_warp_bwd_coarse_kernel<<<grid_1d((size_t)B * S3N_GG, 128), 128, 0, s>>>(fine, dgrid, B, Ho, Wo);
  HK_LAUNCH_CHECK("s3n_warp_bwd_coarse_kernel");
  return 0;
}

int hk_stem_dgrad(const float* dc, const float* w, float* dx, int N, int H, int W, void* stream) {
  HK_REQUIRE(dc && w && dx, HK_ERR_ARG, "hk_stem_dgrad: null pointer");
  HK_REQUIRE(N > 0 && H > 0 && W > 0, HK_ERR_ARG, "hk_stem_dgrad: N=%d H=%d W=%d", N, H, W);
  HK_REQUIRE(aligned16(dc), HK_ERR_ALIGN, "hk_stem_dgrad: dc must be 16-byte aligned");
  const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
  stem_dgrad_kernel<<<grid_1d((size_t)N * H * W, 256), 256, 0, (cudaStream_t)stream>>>(dc, w, dx, N, H, W, Ho, Wo);
  HK_LAUNCH_CHECK("stem_dgrad_kernel");
  return 0;
}

}  // extern "C"
