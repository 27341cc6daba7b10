// VGG-16 backbone convolutions (reference model/backbone/vgg.py:56-70: Conv2d 3x3 s1 p1 + bias, ReLU,
// MaxPool2d 2x2) as im2col-free implicit GEMMs on wgmma (tf32 inputs, fp32 accumulate in registers).
//
// Layout: activations are NHWC fp32 inside the backbone.  For a 3x3 tap (kh,kw) the A operand of the
// implicit GEMM is the input window shifted by (kh-1,kw-1); a 4-D TMA box {32 ch, TW, TH, TN} at the
// shifted (possibly negative) coordinate lands as 128 rows x 128 B in 128B-swizzled shared memory —
// exactly the K-major wgmma operand layout — and TMA's out-of-bounds zero fill *is* the conv padding.
//   fwd   : Y[pix, co]  = sum_{tap,ci} X[pix+tap, ci] * Wf[tap][co][ci]        (+bias, ReLU)
//   dgrad : dX[pix, ci] = sum_{tap,co} dY[pix+tap, co] * Wd[tap][ci][co]       (Wd = flipped/transposed W; * (act>0))
//   wgrad : dW[tap][ci][co] = sum_pix X[pix+tap, ci] * dY[pix, co]             (X in registers, dY^T in smem; split-K)
#include <stdlib.h>

#include "common.cuh"
#include "host.h"
#include "gemm.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

// ------------------------------------------------------------------------------------------------
// weight packing:  W [Cout][Cin][3][3]  ->  Wf [9][Cout][Cin]  and  Wd [9][Cin][Cout] (taps flipped)
// ------------------------------------------------------------------------------------------------
__global__ void pack_weights_kernel(const float* __restrict__ W, float* __restrict__ Wf, float* __restrict__ Wd,
                                    int Cout, int Cin, int round) {
  const size_t n = (size_t)Cout * Cin * 9;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int t = i % 9;
    const int ci = (i / 9) % Cin;
    const int co = i / ((size_t)9 * Cin);
    const float v = round ? tf32_round(W[i]) : W[i];
    if (Wf) Wf[((size_t)t * Cout + co) * Cin + ci] = v;
    if (Wd) Wd[((size_t)(8 - t) * Cin + ci) * Cout + co] = v;
  }
}
// dWp [9][Cin][Cout] -> dW [Cout][Cin][3][3]
__global__ void unpack_wgrad_kernel(const float* __restrict__ dWp, float* __restrict__ dW, int Cout, int Cin, int accumulate) {
  const size_t n = (size_t)Cout * Cin * 9;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int t = i % 9;
    const int ci = (i / 9) % Cin;
    const int co = i / ((size_t)9 * Cin);
    const float v = dWp[((size_t)t * Cin + ci) * Cout + co];
    dW[i] = accumulate ? dW[i] + v : v;
  }
}

// ------------------------------------------------------------------------------------------------
// implicit-GEMM conv (forward and data-gradient)
// ------------------------------------------------------------------------------------------------
struct ConvArgs {
  float* Y;            // [N,H,W,Cout]
  const float* bias;   // [Cout] or null
  const float* mask;   // [N,H,W,Cout] or null: out *= (mask > 0)   (ReLU backward fused into dgrad)
  int N, H, W, Cin, Cout;
  int TW, TH, TN;      // pixel tile (product 128)
  int tiles_w, tiles_h, tiles_n;
  int relu;
  int stride;          // 1 or 2 (N,H,W above are OUTPUT dims; the input map is H*stride x W*stride)
  const float* addend; // [N,H,W,Cout] or null: raw partial sum added to the accumulator first (3xTF32 passes; may alias Y)
  int no_round;        // 1: store fp32 as is (precise mode); 0: round to tf32 (the output feeds another MMA)
  // fused MaxPool2d(2,2) epilogue (vgg.py:59): when P != null the full-resolution map Y is NOT written; the epilogue
  // reduces each 2x2 window (the generic kernel across lanes: the pixel tile is a power-of-two patch, so the window
  // partners are lane^1, lane^TW, lane^(TW+1); the v2 kernel in its staging tile) and writes the pooled value plus, if
  // code != null, the byte maxpool2x2_bwd_idx reads (bits 0-1 = first maximum in scan order, bit 2 = max > 0).
  float* P;            // [N,H/2,W/2,Cout] (or [N,Cout,H/2,W/2] when pool_nchw)
  unsigned char* code; // [N,H/2,W/2,Cout] or null.  EPI_UNPOOL reads it instead: [N,H,W,Cout], and Y is [N,2H,2W,Cout]
  int pool_nchw;
};

// 2x2 max-pool of one 32-channel chunk held as v[32] by the thread of pixel (w, h): window partners are lanes ^1, ^TW and
// ^(TW|1).  Written by the top-left lane of each window.  Bit-identical to maxpool2x2_fwd_idx_kernel on the stored map.
__device__ __forceinline__ void epi_pool_store(const ConvArgs& a, const float* v, int TW, int w, int h, int n, int co,
                                               bool valid) {
  const bool writer = valid && !(w & 1) && !(h & 1);
  const int Ho = a.H >> 1, Wo = a.W >> 1;
  const size_t pp = ((size_t)n * Ho + (h >> 1)) * Wo + (w >> 1);
  float m[32];
  unsigned char cd[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float v0 = v[j];
    const float v1 = __shfl_xor_sync(0xffffffffu, v0, 1);
    const float v2 = __shfl_xor_sync(0xffffffffu, v0, TW);
    const float v3 = __shfl_xor_sync(0xffffffffu, v0, TW | 1);
    float mm = v0;
    unsigned char k = 0;
    if (v1 > mm) { mm = v1; k = 1; }
    if (v2 > mm) { mm = v2; k = 2; }
    if (v3 > mm) { mm = v3; k = 3; }
    m[j] = mm;
    cd[j] = k | (mm > 0.f ? 4 : 0);
  }
  if (!writer) return;
  if (a.code) {
    uint32_t pk[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      pk[j] = (uint32_t)cd[4 * j] | ((uint32_t)cd[4 * j + 1] << 8) | ((uint32_t)cd[4 * j + 2] << 16) | ((uint32_t)cd[4 * j + 3] << 24);
    uint4* cp = reinterpret_cast<uint4*>(a.code + pp * a.Cout + co);
    cp[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    cp[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
  }
  if (!a.pool_nchw) {
    float4* dst = reinterpret_cast<float4*>(a.P + pp * a.Cout + co);
#pragma unroll
    for (int j = 0; j < 8; ++j) dst[j] = make_float4(m[4 * j], m[4 * j + 1], m[4 * j + 2], m[4 * j + 3]);
  } else {
    const size_t hw = (size_t)Ho * Wo;
    float* dst = a.P + ((size_t)n * a.Cout + co) * hw + (size_t)(h >> 1) * Wo + (w >> 1);
#pragma unroll
    for (int j = 0; j < 32; ++j) dst[(size_t)j * hw] = m[j];
  }
}

constexpr int CONV_THREADS = 384;

template <int BN>
struct ConvCfg {
  static constexpr int STAGES = 4;
  static constexpr int A_BYTES = 128 * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_TILE = 2 * 128 * 33 * 4;   // two 32-column accumulator chunks, row-major, padded rows
  static constexpr int SMEM = STAGES * STAGE_BYTES + 1024 + 256 + ACC_TILE;
};

// Output of one 32-column chunk v (channels co .. co + 31) of pixel (w, h, n): addend, bias, ReLU, mask, then the stored
// map or the fused pooling.  Every lane of the warp calls it (the pooling shuffles are warp-wide), valid or not; lane
// 32 q + l must hold pixel r = 32 q + l of the tile.  POOLED: the caller knows that a.P is set, and
// with it neither addend nor mask (the fused pooling belongs to the single-pass forward).
template <bool POOLED = false>
__device__ __forceinline__ void epi_chunk(const ConvArgs& a, float (&v)[32], int w, int h, int n, size_t pix, int co,
                                          bool valid) {
  if (valid && co < a.Cout) {
    if (!POOLED && a.addend) {
      const float4* ad = reinterpret_cast<const float4*>(a.addend + pix * a.Cout + co);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 t = ad[j];
        v[4 * j] += t.x; v[4 * j + 1] += t.y; v[4 * j + 2] += t.z; v[4 * j + 3] += t.w;
      }
    }
    if (a.bias) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] += __ldg(a.bias + co + j);
    }
    if (a.relu) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
    }
    if (!POOLED && a.mask) {
      const float4* m = reinterpret_cast<const float4*>(a.mask + pix * a.Cout + co);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 mm = __ldcs(m + j);   // read once: must not displace the operands the main loop re-reads from L2
        v[4 * j] = mm.x > 0.f ? v[4 * j] : 0.f;
        v[4 * j + 1] = mm.y > 0.f ? v[4 * j + 1] : 0.f;
        v[4 * j + 2] = mm.z > 0.f ? v[4 * j + 2] : 0.f;
        v[4 * j + 3] = mm.w > 0.f ? v[4 * j + 3] : 0.f;
      }
    }
    if (POOLED || a.P) {       // (never combined with the precise-mode passes: rounded like the stored map would be)
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = tf32_round(v[j]);
    } else {
    float4* dst = reinterpret_cast<float4*>(a.Y + pix * a.Cout + co);
    if (a.no_round) {
#pragma unroll
      for (int j = 0; j < 8; ++j) dst[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        dst[j] = make_float4(tf32_round(v[4 * j]), tf32_round(v[4 * j + 1]), tf32_round(v[4 * j + 2]),
                             tf32_round(v[4 * j + 3]));
    }
    }
  }
  // the window reduction is a warp-wide shuffle: every lane takes part, whether or not its own pixel is valid
  if ((POOLED || a.P) && co < a.Cout) epi_pool_store(a, v, a.TW, w, h, n, co, valid);
}

// Epilogue of one 128-pixel x BN tile, run by the 256 MMA threads (ct = thread index among them).  The accumulators go
// through shared memory two 32-column chunks at a time, after which thread (half, q, lane) owns pixel r = 32 q + lane of
// chunk 2 c + half — the mapping the fused pooling shuffles rely on.
template <int BN>
__device__ __forceinline__ void conv_epilogue(const ConvArgs& a, const float (&acc)[BN / 2], float* acc_tile, int w0, int h0,
                                              int n0, int co0, int ct) {
  constexpr int NACC = BN / 2;
  const int lane = ct & 31, wg = ct >> 7, half = ct >> 7;
  const int q = (ct >> 5) & 3, wl = q;
  const int r = q * 32 + lane;
  const int wi = r % a.TW, hi = (r / a.TW) % a.TH, ni = r / (a.TW * a.TH);
  const int w = w0 + wi, h = h0 + hi, n = n0 + ni;
  const bool valid = (w < a.W) && (h < a.H) && (n < a.N);
  const size_t pix = ((size_t)n * a.H + h) * a.W + w;
#pragma unroll
  for (int cp = 0; cp < BN / 64; ++cp) {
    named_bar(1, 256);
#pragma unroll
    for (int i = 0; i < NACC / 4; ++i) {
      const int col = 8 * i + 2 * (lane & 3);
      if ((col >> 6) != cp) continue;
      float* dst = acc_tile + ((col >> 5) & 1) * (128 * 33);
      const int r0 = wg * 64 + wl * 16 + (lane >> 2);
      dst[r0 * 33 + (col & 31)] = acc[4 * i];
      dst[r0 * 33 + (col & 31) + 1] = acc[4 * i + 1];
      dst[(r0 + 8) * 33 + (col & 31)] = acc[4 * i + 2];
      dst[(r0 + 8) * 33 + (col & 31) + 1] = acc[4 * i + 3];
    }
    named_bar(1, 256);
    const int c = 2 * cp + half;
    float v[32];
    {
      const float* src = acc_tile + half * (128 * 33) + r * 33;
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = src[j];
    }
    epi_chunk(a, v, w, h, n, pix, co0 + c * 32, valid);
  }
}

// warpgroup 0: TMA producer (one thread); warpgroups 1-2: wgmma on rows 0-63 / 64-127 of the 128-pixel tile, then the
// epilogue.  The accumulators go through shared memory two 32-column chunks at a time, after which consumer thread
// (half, q, lane) owns pixel r = 32 q + lane of chunk 2 c + half — the mapping the fused pooling shuffles rely on.
template <int BN>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv3x3_igemm_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, ConvArgs a) {
  using Cfg = ConvCfg<BN>;
  constexpr int NACC = BN / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + Cfg::STAGES * Cfg::A_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty = full + Cfg::STAGES;
  float* acc_tile = reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES + 256);

  const int warp = threadIdx.x >> 5;
  int t = blockIdx.x;
  const int tw = t % a.tiles_w; t /= a.tiles_w;
  const int th = t % a.tiles_h; t /= a.tiles_h;
  const int w0 = tw * a.TW, h0 = th * a.TH, n0 = t * a.TN;
  const int co0 = blockIdx.y * BN;
  const int nchunk = a.Cin / 32;
  const int nk = 9 * nchunk;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    regs_dealloc<56>();
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < nk; ++kb) {
        const int s = kb % Cfg::STAGES;
        const uint32_t ph = (kb / Cfg::STAGES) & 1;
        const int tap = kb / nchunk, ck = kb - tap * nchunk;
        const int kh = tap / 3, kw = tap - kh * 3;
        mbar_wait(&empty[s], ph ^ 1);
        mbar_expect_tx(&full[s], Cfg::STAGE_BYTES);
        tma_load_4d(sA + s * Cfg::A_BYTES, &tmX, &full[s], ck * 32, w0 * a.stride + kw - 1, h0 * a.stride + kh - 1, n0);
        tma_load_3d(sB + s * Cfg::B_BYTES, &tmW, &full[s], ck * 32, co0, tap);
      }
    }
  } else {
    regs_alloc<224>();
    const int ct = threadIdx.x - 128;
    const int wg = ct >> 7;
    float acc[NACC];          // overwritten by the first MMA (scale-d = 0): nk >= 9
    for (int kb = 0; kb < nk; ++kb) {
      const int s = kb % Cfg::STAGES;
      const uint32_t ph = (kb / Cfg::STAGES) & 1;
      mbar_wait(&full[s], ph);
      const uint64_t a_base = make_sdesc(smem_u32(sA + s * Cfg::A_BYTES + wg * 64 * 128));
      const uint64_t b_base = make_sdesc(smem_u32(sB + s * Cfg::B_BYTES));
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) wgmma_tf32(acc, a_base + ks * 2, b_base + ks * 2, (kb | ks) != 0);
      wgmma_commit();
      wgmma_wait<1>();          // k-block kb stays in flight; the stage of kb - 1 is free
      wgmma_keep(acc);
      if (kb > 0 && (ct & 127) == 0) mbar_arrive(&empty[(kb - 1) % Cfg::STAGES]);
    }
    wgmma_wait<0>();
    wgmma_keep(acc);
    conv_epilogue<BN>(a, acc, acc_tile, w0, h0, n0, co0, ct);
  }
}

// pick a pixel tile TW x TH x TN with product `target` that tiles W x H (x N) with as little waste as possible
static void pick_tile(int W, int H, int N, int target, int* TW, int* TH, int* TN) {
  int tw = 1;
  while (tw * 2 <= 16 && W % (tw * 2) == 0 && tw * 2 <= target) tw *= 2;
  int th = 1;
  while (th * 2 * tw <= target && H % (th * 2) == 0) th *= 2;
  int tn = target / (tw * th);
  // if the map is tiny (e.g. 2x2) the remainder goes to the batch dimension
  *TW = tw; *TH = th; *TN = tn;
  (void)N;
}

static int make_act_map(CUtensorMap* tm, const float* X, int N, int H, int W, int C, int TW, int TH, int TN,
                        int stride = 1) {
  uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)N};
  uint64_t strides[3] = {(uint64_t)C * 4, (uint64_t)W * C * 4, (uint64_t)H * W * C * 4};
  // strided traversal: the box spans TW*stride elements and TMA keeps every stride-th one
  uint32_t box[4] = {32, (uint32_t)(TW * stride), (uint32_t)(TH * stride), (uint32_t)TN};
  uint32_t estr[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
  return make_tmap(tm, X, 4, dims, strides, box, stride > 1 ? estr : nullptr);
}

template <int BN>
static int launch_conv(const CUtensorMap& tmX, const CUtensorMap& tmW, const ConvArgs& a, cudaStream_t stream) {
  using Cfg = ConvCfg<BN>;
  if (int r = allow_dynamic_smem<conv3x3_igemm_kernel<BN>>(Cfg::SMEM, BN == 64 ? "conv<64>" : "conv<128>")) return r;
  dim3 grid(a.tiles_w * a.tiles_h * a.tiles_n, (a.Cout + BN - 1) / BN);
  conv3x3_igemm_kernel<BN><<<grid, CONV_THREADS, Cfg::SMEM, stream>>>(tmX, tmW, a);
  HK_LAUNCH_CHECK("conv3x3_igemm_kernel");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// implicit-GEMM conv v2 (stride 1, maps with W % 8 == 0 and H % 8 == 0): persistent CTAs and halo reuse.
//   * pixel tile (M = 128): 16 wide x 8 high of one image where 16 divides W, else 8 x 8 of two consecutive images (the
//     56 x 56 maps; an odd batch leaves the last tile's second image empty: TMA zero-fills it, the epilogue skips it).
//     For each (cin chunk, kw) ONE TMA load brings the (8+2)-row halo patch of every image of the tile (160 rows x
//     128 B); the three kh taps are the same patch addressed kh*TW rows (2 KB / 1 KB = whole swizzle atoms) further down,
//     so the input crosses the L2->SM fabric 3x (+25 % halo) instead of 9x.  MMA warpgroup wg takes rows 64 wg.. of the
//     tile: the lower half of the 16 x 8 patch, or image wg of the pair (its patch starts 80 rows = 10 atoms down).
//   * RESIDENT (Cin = 64, Cout = 64: VGG conv1_2 and its dgrad): all 9x2 weight tiles (144 KB) stay in shared memory for
//     the life of the CTA; only activations stream.
//   * the shared-memory ring runs across tiles, so the producer loads tile i+1 while the MMA warpgroups finish tile i.
//   * BN = 128 has room for two 68 KB stages beside the staging tile, which is too shallow to hide a stage's load: with
//     the epilogue removed the forward main loop ran at 295-310 TFLOP/s, at 340-360 when the weights were loaded only for
//     a CTA's first tile, and at 380-420 with a third stage in place of the staging tile (H100 SXM, 700 W).  So the bound
//     is the latency of a stage's load, not the bytes it moves (two-CTA clusters that multicast each weight tile, 35 %
//     fewer L2 bytes per stage, ran at ~200 TFLOP/s: a slot is freed only when both CTAs have released it), and each
//     stage there
//     has three full barriers, {halo patch + kh 0 weights, kh 1 weights, kh 2 weights}, and one wgmma group per piece:
//     the MMAs of a piece start as soon as it has landed, and the previous stage is handed back after the first group
//     is issued, while the later pieces may still be in flight.  The accumulation order does not change.  The BN = 64
//     ring is three stages deep and keeps one barrier per stage.
//   * the MMA warpgroups hand each finished tile to a fourth, epilogue warpgroup through a shared-memory staging tile and
//     go straight on to the next tile: the output stores and the mask loads of tile i overlap the MMAs of tile i+1.
//   * the epilogue of the stored map has 8 lanes per pixel (one float4 of the 32-channel chunk each), so a warp's load
//     or store instruction covers 4 whole 128-byte lines (with thread = pixel it touched 32 lines, 16 bytes of each).
//     Mask loads and output stores are streaming (ld.global.cs / st.global.cs): each byte is touched once, and as
//     ordinary accesses the mask pushed the halo rows and weight tiles that neighbouring CTAs re-read out of L2, which
//     cost the data gradient of the 128-channel-and-deeper layers 8-20 %.  Asking
//     for the mask a chunk ahead of its use measured no different and is not done.  The fused pooling keeps thread =
//     pixel, which its shuffles need.
// ------------------------------------------------------------------------------------------------
constexpr int CONV_V2_THREADS = 512;

// what the epilogue warpgroup of the stored map does with a finished tile (the fused pooling is selected by ConvArgs::P):
//   EPI_MAP          store it (bias, ReLU, mask, tf32 rounding).
//   EPI_UNPOOL       the data gradient of a layer whose input came from a 2x2 max-pool: round to tf32, keep it where the
//                    pool's byte has bit 2, and store it at window position (code & 3) of the full-resolution map, zeros at
//                    the other three — what maxpool2x2_bwd_idx_kernel does with the stored map, so the bits are the same
//                    and the pooled gradient is never written.
//   EPI_FIRST_WGRAD  the data gradient of VGG conv1_2 (resident 64 -> 64, 16 x 8 tile): mask and round as EPI_MAP, then,
//                    instead of storing dX, accumulate conv1_1's D[co][j] += sum_px dX[px][co] X27[px][j] on mma.sync from
//                    the staging tile and the tile's image halo.  Each CTA writes its D to fw.part at the end.
enum { EPI_MAP = 0, EPI_UNPOOL = 1, EPI_FIRST_WGRAD = 2 };
// EPI_FIRST_WGRAD image halo of one 16 x 8 tile: 3 channels x (8 + 2) rows x (16 + 2) columns, tf32-rounded, zero padded.
// Two buffers (the tile being summed and the next one) beside the resident configuration's 226,560 bytes.
constexpr int FW_HALO = 3 * 10 * 18;
constexpr int FW_HALO_BYTES = 2 * FW_HALO * 4;
struct FirstWgradArgs {
  const float* img;   // the NCHW image conv1_1 read
  float* part;        // [gridDim.x][64][32] partials of conv1_1's dW^T (column 27: db)
};

// D (16 x 8, fp32) += A (16 x 8, tf32, row-major) . B (8 x 8, tf32, column-major)
__device__ __forceinline__ void mma_m16n8k8_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int BN, bool RESIDENT>
struct ConvV2Cfg {
  static constexpr int A_BYTES = 160 * 128;                          // 20 KB halo patch
  static constexpr int B_TILE = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + (RESIDENT ? 0 : 3 * B_TILE);
  static constexpr int STAGES = RESIDENT ? 2 : (BN == 64 ? 3 : 2);
  static constexpr int WRES_BYTES = RESIDENT ? 18 * B_TILE : 0;      // 9 taps x 2 chunks
  // full barriers per stage: {halo patch + kh 0 weights, kh 1 weights, kh 2 weights} where the ring is two stages deep,
  // else one for the whole stage
  static constexpr int PIECES = STAGES == 2 && !RESIDENT ? 3 : 1;
  // staging tile [128 pixels][BN + 8] fp32: the padding makes the MMA threads' 8-byte fragment stores conflict-free
  // (rows 8 words apart in bank space, 4 lanes x 8 B per row); the epilogue of the stored map reads a pixel's 128-byte
  // chunk with 8 consecutive lanes, one float4 each: all 32 banks once per quarter-warp, whatever the pitch.
  static constexpr int STG_LD = BN + 8;
  static constexpr int STG_BYTES = 128 * STG_LD * 4;
  static constexpr int SMEM = STAGES * STAGE_BYTES + WRES_BYTES + 1024 + 256 + STG_BYTES;
};

// warpgroup 0: TMA producer (one thread); warpgroups 1-2: wgmma on rows 0-63 / 64-127 of the 128-pixel tile; warpgroup 3:
// the epilogue.  TW = 16: tile 16 x 8 x 1 image, TW = 8: tile 8 x 8 x 2 images.
template <int BN, bool RESIDENT, int TW, int EPI>
__global__ void __launch_bounds__(CONV_V2_THREADS, 1)
conv3x3_igemm_v2_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, ConvArgs a,
                        int n_ntiles, int total_tiles, FirstWgradArgs fw) {
  using Cfg = ConvV2Cfg<BN, RESIDENT>;
  static_assert(EPI != EPI_FIRST_WGRAD || (BN == 64 && RESIDENT && TW == 16), "conv1_1 weight gradient: 64 -> 64, 16 x 8");
  constexpr int NACC = BN / 2;
  constexpr int TN = 16 / TW;                       // images per tile
  constexpr int WG_ROWS = TW == 16 ? 64 : 80;       // patch rows between the two MMA warpgroups' A operands
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stages = smem;
  uint8_t* wres = smem + Cfg::STAGES * Cfg::STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(wres + Cfg::WRES_BYTES);   // [STAGES][PIECES]
  uint64_t* empty = full + Cfg::STAGES * Cfg::PIECES;
  uint64_t* wbar = empty + Cfg::STAGES;
  uint64_t* stg_full = wbar + 1;                    // the MMA threads wrote the staging tile (256 arrivals)
  uint64_t* stg_empty = wbar + 2;                   // the epilogue threads read it (128 arrivals)
  float* stg = reinterpret_cast<float*>(wres + Cfg::WRES_BYTES + 256);

  const int warp = threadIdx.x >> 5;
  const int nchunk = a.Cin / 32;
  const int nkb = nchunk * 3;                       // (chunk, kw) steps per tile

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    for (int s = 0; s < Cfg::STAGES; ++s) mbar_init(&empty[s], 2);
    for (int i = 0; i < Cfg::STAGES * Cfg::PIECES; ++i) mbar_init(&full[i], 1);
    mbar_init(wbar, 1);
    mbar_init(stg_full, 256);
    mbar_init(stg_empty, 128);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 12 && EPI == EPI_MAP && a.P) {
    // fused pooling: thread r owns pixel r of the tile, the mapping epi_chunk's pooling shuffles rely on.  The staging
    // tile is released as soon as its last chunk has been read.
    const int r = threadIdx.x - 384;
    int j = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++j) {
      int pt = t / n_ntiles;
      const int co0 = (t - pt * n_ntiles) * BN;
      const int tw = pt % a.tiles_w; pt /= a.tiles_w;
      const int th = pt % a.tiles_h; pt /= a.tiles_h;
      mbar_wait(stg_full, j & 1);
      const int w = tw * TW + (r & (TW - 1)), h = th * 8 + ((r / TW) & 7), n = pt * TN + r / (TW * 8);
      const bool valid = TN == 1 || n < a.N;
      const size_t pix = ((size_t)n * a.H + h) * a.W + w;
#pragma unroll 1
      for (int c = 0; c < BN / 32; ++c) {
        float v[32];
        const float4* src = reinterpret_cast<const float4*>(stg + r * Cfg::STG_LD + c * 32);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float4 q = src[k];
          v[4 * k] = q.x; v[4 * k + 1] = q.y; v[4 * k + 2] = q.z; v[4 * k + 3] = q.w;
        }
        if (c == BN / 32 - 1) mbar_arrive(stg_empty);
        epi_chunk<true>(a, v, w, h, n, pix, co0 + c * 32, valid);
      }
    }
  } else if (warp >= 12) {
    // stored map (never the precise-mode passes: no addend, always rounded).  Lane (sub, u) = (lane / 8, lane % 8) of warp
    // ew owns channels 4 u .. 4 u + 3 of pixels 32 ew + 4 k + sub, k = 0..7, in every 32-channel chunk.
    const int e = threadIdx.x - 384;
    const int ew = e >> 5, sub = (e >> 3) & 3, u4 = (e & 7) * 4;
    // element offset of pixel k = 0 from the tile origin's first channel; pixel k is k % (TW / 4) steps of 4 pixels and
    // k / (TW / 4) map rows further on
    const int p0 = ew * 32 + sub;
    const int eoff0 = (TW == 16 ? (p0 >> 4) * a.W + (p0 & 15) : ((p0 >> 6) * a.H + ((p0 >> 3) & 7)) * a.W + (p0 & 7)) * a.Cout + u4;
    const int erow = a.W * a.Cout, e4 = 4 * a.Cout;
    auto eoff = [&](int k) { return eoff0 + (k / (TW / 4)) * erow + (k % (TW / 4)) * e4; };
    const float* srow = stg + (ew * 32 + sub) * Cfg::STG_LD + u4;
    // origin element and first channel of tile t; false if this warp's image lies beyond the batch
    auto tile_org = [&](int t, size_t& org, int& co0) {
      co0 = (t % n_ntiles) * BN;
      int pt = t / n_ntiles;
      const int tw = pt % a.tiles_w; pt /= a.tiles_w;
      const int th = pt % a.tiles_h; pt /= a.tiles_h;
      org = (((size_t)pt * TN * a.H + th * 8) * a.W + tw * TW) * a.Cout;
      return pt * TN + (TW == 16 ? 0 : ew >> 1) < a.N;
    };
    // pixel-tile coordinates (column, row, first image) of tile t
    auto tile_pos = [&](int t, int& tw, int& th, int& tn) {
      int pt = t / n_ntiles;
      tw = pt % a.tiles_w; pt /= a.tiles_w;
      th = pt % a.tiles_h; tn = pt / a.tiles_h;
    };
    // EPI_UNPOOL: element offset of pixel k's window (top-left) from the full-resolution tile origin, as eoff
    const int frow = 2 * a.W * a.Cout;
    const int uoff0 = (TW == 16 ? 2 * (p0 >> 4) * frow + 2 * (p0 & 15) * a.Cout
                                : ((p0 >> 6) * 2 * a.H + 2 * ((p0 >> 3) & 7)) * frow + 2 * (p0 & 7) * a.Cout) + u4;
    auto uoff = [&](int k) { return uoff0 + (k / (TW / 4)) * 2 * frow + (k % (TW / 4)) * 8 * a.Cout; };
    // EPI_FIRST_WGRAD.  mma.sync fragments of warp ew, which owns co 16 ew .. 16 ew + 15 and all 32 X27 columns
    // (g = lane / 4, tq = lane % 4): A[co][px] = dX[px][co] is read from the staging tile, rows px = 8 ks + tq (+4),
    // columns 16 ew + g (+8) (the 72-float pitch puts the 32 lanes in 32 banks); B[px][j] = X27[px][j] for column
    // j = 8 nt + g is halo element hoff[nt] + (px / 16) * 18 + px % 16 (j < 27), 1 for j = 27, 0 after.
    float* halo = stg + 128 * Cfg::STG_LD;
    float dacc[4][4] = {};
    const int lane = e & 31, g = lane >> 2, tq = lane & 3;
    int hoff[4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int jj = 8 * nt + g;
      hoff[nt] = jj < 27 ? (jj / 9) * 180 + (jj % 9 / 3) * 18 + jj % 3 : 0;
    }
    int co0 = 0, j = 0;
    size_t org = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++j) {
      const bool valid = tile_org(t, org, co0);
      if constexpr (EPI == EPI_FIRST_WGRAD) {
        // this tile's halo, loaded while the MMA warpgroups are still on it.  Buffer j & 1 was last read for tile j - 2,
        // before every epilogue thread passed tile j - 1's barrier.
        int tw, th, tn;
        tile_pos(t, tw, th, tn);
        float* hb = halo + (j & 1) * FW_HALO;
        for (int i = e; i < FW_HALO; i += 128) {
          const int ci = i / 180, hh = th * 8 - 1 + i / 18 % 10, ww = tw * 16 - 1 + i % 18;
          hb[i] = hh >= 0 && hh < a.H && ww >= 0 && ww < a.W
                      ? tf32_round(__ldg(fw.img + (((size_t)tn * 3 + ci) * a.H + hh) * a.W + ww)) : 0.f;
        }
      }
      mbar_wait(stg_full, j & 1);
#pragma unroll
      for (int c = 0; c < BN / 32; ++c) {
        float4 v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = *reinterpret_cast<const float4*>(srow + 4 * k * Cfg::STG_LD + c * 32);
        if (EPI != EPI_FIRST_WGRAD && c == BN / 32 - 1) mbar_arrive(stg_empty);
        const int co = co0 + c * 32;
        const bool live = valid && co < a.Cout;
        if (live) {
          if (a.bias) {
            const float4 b = __ldg(reinterpret_cast<const float4*>(a.bias + co + u4));
#pragma unroll
            for (int k = 0; k < 8; ++k) { v[k].x += b.x; v[k].y += b.y; v[k].z += b.z; v[k].w += b.w; }
          }
          if (a.relu) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              v[k].x = fmaxf(v[k].x, 0.f); v[k].y = fmaxf(v[k].y, 0.f);
              v[k].z = fmaxf(v[k].z, 0.f); v[k].w = fmaxf(v[k].w, 0.f);
            }
          }
          if (a.mask) {
            float4 mk[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) mk[k] = __ldcs(reinterpret_cast<const float4*>(a.mask + org + co + eoff(k)));
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              v[k].x = mk[k].x > 0.f ? v[k].x : 0.f; v[k].y = mk[k].y > 0.f ? v[k].y : 0.f;
              v[k].z = mk[k].z > 0.f ? v[k].z : 0.f; v[k].w = mk[k].w > 0.f ? v[k].w : 0.f;
            }
          }
          if constexpr (EPI == EPI_MAP) {
#pragma unroll
            for (int k = 0; k < 8; ++k)
              __stcs(reinterpret_cast<float4*>(a.Y + org + co + eoff(k)),
                     make_float4(tf32_round(v[k].x), tf32_round(v[k].y), tf32_round(v[k].z), tf32_round(v[k].w)));
          } else if constexpr (EPI == EPI_UNPOOL) {
            int tw, th, tn;
            tile_pos(t, tw, th, tn);
            float* dst = a.Y + (((size_t)tn * TN * 2 * a.H + th * 16) * 2 * a.W + tw * 2 * TW) * a.Cout + co;
            // the four codes of a float4 as one word (byte i: channel i)
            uint32_t cd[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) cd[k] = __ldcs(reinterpret_cast<const unsigned int*>(a.code + org + co + eoff(k)));
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              const float4 q = make_float4((cd[k] & 4u) ? tf32_round(v[k].x) : 0.f, (cd[k] & (4u << 8)) ? tf32_round(v[k].y) : 0.f,
                                           (cd[k] & (4u << 16)) ? tf32_round(v[k].z) : 0.f,
                                           (cd[k] & (4u << 24)) ? tf32_round(v[k].w) : 0.f);
              float* o = dst + uoff(k);
#pragma unroll
              for (int pos = 0; pos < 4; ++pos)
                __stcs(reinterpret_cast<float4*>(o + (pos >> 1) * frow + (pos & 1) * a.Cout),
                       make_float4((cd[k] & 3u) == (uint32_t)pos ? q.x : 0.f, (cd[k] >> 8 & 3u) == (uint32_t)pos ? q.y : 0.f,
                                   (cd[k] >> 16 & 3u) == (uint32_t)pos ? q.z : 0.f,
                                   (cd[k] >> 24 & 3u) == (uint32_t)pos ? q.w : 0.f));
            }
          } else {
            // dX goes back into the staging tile, where the MMAs below read it
#pragma unroll
            for (int k = 0; k < 8; ++k)
              *reinterpret_cast<float4*>(stg + (ew * 32 + sub + 4 * k) * Cfg::STG_LD + u4 + c * 32) =
                  make_float4(tf32_round(v[k].x), tf32_round(v[k].y), tf32_round(v[k].z), tf32_round(v[k].w));
          }
        }
      }
      if constexpr (EPI == EPI_FIRST_WGRAD) {
        named_bar(1, 128);    // the whole of dX and the halo are in shared memory
        const float* hb = halo + (j & 1) * FW_HALO;
        const float* arow = stg + tq * Cfg::STG_LD + 16 * ew + g;
#pragma unroll 4
        for (int ks = 0; ks < 16; ++ks) {
          const float* ap = arow + 8 * ks * Cfg::STG_LD;
          const uint32_t af[4] = {__float_as_uint(ap[0]), __float_as_uint(ap[8]), __float_as_uint(ap[4 * Cfg::STG_LD]),
                                  __float_as_uint(ap[4 * Cfg::STG_LD + 8])};
          const int hp = (ks >> 1) * 18 + 8 * (ks & 1) + tq;    // halo offset of pixel 8 ks + tq
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            float b0 = hb[hoff[nt] + hp], b1 = hb[hoff[nt] + hp + 4];
            if (nt == 3 && g >= 3) b0 = b1 = g == 3 ? 1.f : 0.f;
            mma_m16n8k8_tf32(dacc[nt], af, __float_as_uint(b0), __float_as_uint(b1));
          }
        }
        mbar_arrive(stg_empty);
      }
    }
    if constexpr (EPI == EPI_FIRST_WGRAD) {
      // accumulator i of n-tile nt: co 16 ew + g (+8 for i >= 2), column 8 nt + 2 tq + (i & 1)
      float* dst = fw.part + (size_t)blockIdx.x * 64 * 32;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) dst[(16 * ew + g + 8 * (i >> 1)) * 32 + 8 * nt + 2 * tq + (i & 1)] = dacc[nt][i];
    }
  } else if (warp < 4) {
    if (threadIdx.x == 0) {
      if (RESIDENT) {   // whole filter bank (n_ntiles == 1 by construction): 18 tiles of [BN x 32]
        mbar_expect_tx(wbar, Cfg::WRES_BYTES);
        for (int tap = 0; tap < 9; ++tap)
          for (int ck = 0; ck < 2; ++ck) tma_load_3d(wres + (tap * 2 + ck) * Cfg::B_TILE, &tmW, wbar, ck * 32, 0, tap);
      }
      int kbg = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int nt = t % n_ntiles;
        int pt = t / n_ntiles;
        const int tw = pt % a.tiles_w; pt /= a.tiles_w;
        const int th = pt % a.tiles_h; pt /= a.tiles_h;
        const int w0 = tw * TW, h0 = th * 8, n0 = pt * TN, co0 = nt * BN;
        for (int kb = 0; kb < nkb; ++kb, ++kbg) {
          const int s = kbg % Cfg::STAGES;
          const uint32_t ph = (kbg / Cfg::STAGES) & 1;
          const int ck = kb / 3, kw = kb - ck * 3;
          mbar_wait(&empty[s], ph ^ 1);
          uint64_t* f = full + s * Cfg::PIECES;
          uint8_t* st = stages + s * Cfg::STAGE_BYTES;
          mbar_expect_tx(&f[0], Cfg::PIECES == 3 ? Cfg::A_BYTES + Cfg::B_TILE : Cfg::STAGE_BYTES);
          tma_load_4d(st, &tmX, &f[0], ck * 32, w0 + kw - 1, h0 - 1, n0);
          if (!RESIDENT) {
#pragma unroll
            for (int kh = 0; kh < 3; ++kh) {
              uint64_t* fk = &f[Cfg::PIECES == 3 ? kh : 0];
              if (Cfg::PIECES == 3 && kh > 0) mbar_expect_tx(fk, Cfg::B_TILE);
              tma_load_3d(st + Cfg::A_BYTES + kh * Cfg::B_TILE, &tmW, fk, ck * 32, co0, kh * 3 + kw);
            }
          }
        }
      }
    }
  } else {
    const int ct = threadIdx.x - 128;
    const int wg = ct >> 7;
    if (RESIDENT) mbar_wait(wbar, 0);
    // the first MMA of every tile overwrites the accumulators (scale-d = 0): no register writes inside the wgmma pipeline
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    // this thread's accumulator fragment in the staging tile: rows r0 and r0 + 8, columns 8 i + 2 (lane & 3) + {0, 1}
    float* frag = stg + (wg * 64 + ((ct >> 5) & 3) * 16 + ((ct & 31) >> 2)) * Cfg::STG_LD + 2 * (ct & 3);
    int kbg = 0, j = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++j) {
      for (int kb = 0; kb < nkb; ++kb, ++kbg) {
        const int s = kbg % Cfg::STAGES;
        const int ck = kb / 3, kw = kb - ck * 3;
        const uint32_t ph = (kbg / Cfg::STAGES) & 1;
        // rows 64 wg.. of the tile in the patch of tap kh: + (WG_ROWS wg + TW kh) rows of 128 B
        const uint32_t a_addr = smem_u32(stages + s * Cfg::STAGE_BYTES) + wg * WG_ROWS * 128;
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
          // each piece of the stage is consumed as soon as it has landed, one wgmma group per piece
          if (kh < Cfg::PIECES) {
            mbar_wait(&full[s * Cfg::PIECES + kh], ph);
            wgmma_fence();
          }
          const uint32_t b_addr = RESIDENT ? smem_u32(wres + ((kh * 3 + kw) * 2 + ck) * Cfg::B_TILE)
                                           : smem_u32(stages + s * Cfg::STAGE_BYTES + Cfg::A_BYTES + kh * Cfg::B_TILE);
          const uint64_t ad = make_sdesc(a_addr + kh * TW * 128), bd = make_sdesc(b_addr);
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) wgmma_tf32(acc, ad + ks * 2, bd + ks * 2, (kb | kh | ks) != 0);
          if (kh >= 3 - Cfg::PIECES) wgmma_commit();
          if (kh == 3 - Cfg::PIECES) {
            // the first group of step kb stays in flight; the stage of the previous step is free, and is handed back
            // while this step's later pieces may still be landing
            wgmma_wait<1>();
            wgmma_keep(acc);
            if (kb > 0 && (ct & 127) == 0) mbar_arrive(&empty[(kbg - 1) % Cfg::STAGES]);
          }
        }
      }
      wgmma_wait<0>();
      wgmma_keep(acc);
      if ((ct & 127) == 0) mbar_arrive(&empty[(kbg - 1) % Cfg::STAGES]);
      mbar_wait(stg_empty, (j & 1) ^ 1);    // the epilogue warpgroup has read the previous tile
#pragma unroll
      for (int i = 0; i < NACC / 4; ++i) {
        *reinterpret_cast<float2*>(frag + 8 * i) = make_float2(acc[4 * i], acc[4 * i + 1]);
        *reinterpret_cast<float2*>(frag + 8 * Cfg::STG_LD + 8 * i) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
      }
      mbar_arrive(stg_full);
    }
  }
}

template <int BN, bool RESIDENT, int TW, int EPI = EPI_MAP>
static int launch_conv_v2(const float* x, const float* wp, ConvArgs a, int N, int H, int W, cudaStream_t stream,
                          FirstWgradArgs fw = {}) {
  using Cfg = ConvV2Cfg<BN, RESIDENT>;
  constexpr int SMEM = Cfg::SMEM + (EPI == EPI_FIRST_WGRAD ? FW_HALO_BYTES : 0);
  static_assert(SMEM <= 232448, "conv_v2: dynamic shared memory above the sm_90 opt-in limit");
  if (int r = allow_dynamic_smem<conv3x3_igemm_v2_kernel<BN, RESIDENT, TW, EPI>>(SMEM, BN == 64 ? "conv_v2<64>" : "conv_v2<128>"))
    return r;
  a.TW = TW; a.TH = 8; a.TN = 16 / TW;
  a.tiles_w = W / TW; a.tiles_h = H / 8; a.tiles_n = (N + a.TN - 1) / a.TN;
  const int n_ntiles = (a.Cout + BN - 1) / BN;
  const long long total = (long long)a.tiles_w * a.tiles_h * a.tiles_n * n_ntiles;
  HK_REQUIRE(total < (1ll << 31), HK_ERR_UNSUPPORTED, "conv3x3: too many tiles");
  // the epilogue keeps element offsets inside a tile (up to one image apart) as int
  HK_REQUIRE((long long)H * W * a.Cout < (1ll << 30), HK_ERR_UNSUPPORTED, "conv3x3: map too large");
  CUtensorMap tmX, tmW;
  int r;
  {
    uint64_t dims[4] = {(uint64_t)a.Cin, (uint64_t)W, (uint64_t)H, (uint64_t)N};
    uint64_t strides[3] = {(uint64_t)a.Cin * 4, (uint64_t)W * a.Cin * 4, (uint64_t)H * W * a.Cin * 4};
    uint32_t box[4] = {32, (uint32_t)TW, 10, (uint32_t)a.TN};
    if ((r = make_tmap(&tmX, x, 4, dims, strides, box))) return r;
  }
  {
    uint64_t dims[3] = {(uint64_t)a.Cin, (uint64_t)a.Cout, 9};
    uint64_t strides[2] = {(uint64_t)a.Cin * 4, (uint64_t)a.Cin * a.Cout * 4};
    uint32_t box[3] = {32, (uint32_t)BN, 1};
    if ((r = make_tmap(&tmW, wp, 3, dims, strides, box))) return r;
  }
  const int sms = num_sms();
  const int grid = total < sms ? (int)total : sms;
  conv3x3_igemm_v2_kernel<BN, RESIDENT, TW, EPI><<<grid, CONV_V2_THREADS, SMEM, stream>>>(tmX, tmW, a, n_ntiles, (int)total, fw);
  HK_LAUNCH_CHECK("conv3x3_igemm_v2_kernel");
  return 0;
}

template <int TW, int EPI = EPI_MAP>
static int launch_conv_v2(const float* x, const float* wp, const ConvArgs& a, int N, int H, int W, cudaStream_t stream) {
  if (a.Cin == 64 && a.Cout == 64) return launch_conv_v2<64, true, TW, EPI>(x, wp, a, N, H, W, stream);
  if (a.Cout <= 64) return launch_conv_v2<64, false, TW, EPI>(x, wp, a, N, H, W, stream);
  return launch_conv_v2<128, false, TW, EPI>(x, wp, a, N, H, W, stream);
}

static int conv3x3_igemm_1x(const float* x, const float* wp, const float* bias, const float* mask, const float* addend,
                            float* y, int N, int H, int W, int Cin, int Cout, int relu, cudaStream_t stream, int stride,
                            int no_round, float* pooled = nullptr, unsigned char* code = nullptr,
                            int pool_nchw = 0);

// x NHWC [N,H,W,Cin], wp packed [9][Cout][Cin] -> y NHWC [N,H,W,Cout]
int conv3x3_igemm(const float* x, const float* wp, const float* bias, const float* mask, float* y, int N, int H, int W,
                  int Cin, int Cout, int relu, cudaStream_t stream, int stride = 1) {
  if (!precise()) return conv3x3_igemm_1x(x, wp, bias, mask, nullptr, y, N, H, W, Cin, Cout, relu, stream, stride, 0);
  // 3xTF32: y = epi(Xh*Wh + Xl*Wh + Xh*Wl), three passes of the same implicit-GEMM kernel chained through `addend`
  HK_REQUIRE(x && wp && y, HK_ERR_ARG, "conv3x3: null pointer");
  const size_t nx = (size_t)N * H * W * Cin, nw = (size_t)9 * Cout * Cin;
  Scratch sx(2 * nx * sizeof(float), stream), sw(2 * nw * sizeof(float), stream);
  HK_REQUIRE(sx.p && sw.p, HK_ERR_DRIVER, "conv3x3 (precise): cudaMallocAsync of the operand halves failed");
  float *xh = sx.f(), *xl = xh + nx, *wh = sw.f(), *wl = wh + nw;
  int r;
  if ((r = tf32_split(x, xh, xl, nx, stream))) return r;
  if ((r = tf32_split(wp, wh, wl, nw, stream))) return r;
  if ((r = conv3x3_igemm_1x(xh, wl, nullptr, nullptr, nullptr, y, N, H, W, Cin, Cout, 0, stream, stride, 1))) return r;
  if ((r = conv3x3_igemm_1x(xl, wh, nullptr, nullptr, y, y, N, H, W, Cin, Cout, 0, stream, stride, 1))) return r;
  return conv3x3_igemm_1x(xh, wh, bias, mask, y, y, N, H, W, Cin, Cout, relu, stream, stride, 1);
}

static int conv3x3_igemm_1x(const float* x, const float* wp, const float* bias, const float* mask, const float* addend,
                            float* y, int N, int H, int W, int Cin, int Cout, int relu, cudaStream_t stream, int stride,
                            int no_round, float* pooled, unsigned char* code, int pool_nchw) {
  // H, W are the INPUT dims; output is H/stride x W/stride (padding 1)
  const int Hin = H, Win = W;
  if (stride == 2) {
    HK_REQUIRE(H % 2 == 0 && W % 2 == 0, HK_ERR_UNSUPPORTED, "conv3x3 stride 2: even H/W required");
    H /= 2; W /= 2;
  }
  HK_REQUIRE(x && wp && (y || pooled), HK_ERR_ARG, "conv3x3: null pointer");
  HK_REQUIRE(Cin % 32 == 0 && Cout % 32 == 0, HK_ERR_UNSUPPORTED, "conv3x3: Cin=%d Cout=%d must be multiples of 32",
             Cin, Cout);
  HK_REQUIRE(aligned16(x) && aligned16(wp) && (!y || aligned16(y)) && (!mask || aligned16(mask)), HK_ERR_ALIGN,
             "conv3x3: pointer not 16-byte aligned");
  if (pooled)
    HK_REQUIRE(stride == 1 && H % 2 == 0 && W % 2 == 0 && aligned16(pooled) && (!code || aligned16(code)), HK_ERR_UNSUPPORTED,
               "conv3x3 + pool: even H/W, stride 1 and 16-byte aligned outputs required");
  ConvArgs a = {};
  a.P = pooled; a.code = code; a.pool_nchw = pool_nchw;
  a.Y = y; a.bias = bias; a.mask = mask; a.N = N; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.relu = relu;
  a.stride = stride;
  a.addend = addend; a.no_round = no_round;
  // the three chained 3xTF32 passes (no_round) keep the generic kernel, whose accumulation order does not depend on the
  // map size; the single-pass layers take the halo-reuse kernel wherever one of its pixel tiles (16 x 8 x 1 image, else
  // 8 x 8 x 2 images) divides the map
  if (!no_round && stride == 1 && W % 8 == 0 && H % 8 == 0) {
    if (W % 16 == 0) return launch_conv_v2<16>(x, wp, a, N, H, W, stream);
    return launch_conv_v2<8>(x, wp, a, N, H, W, stream);
  }
  pick_tile(W, H, N, 128, &a.TW, &a.TH, &a.TN);
  HK_REQUIRE(!pooled || (a.TW >= 2 && a.TH >= 2), HK_ERR_UNSUPPORTED, "conv3x3 + pool: pixel tile %dx%d", a.TW, a.TH);
  a.tiles_w = (W + a.TW - 1) / a.TW; a.tiles_h = (H + a.TH - 1) / a.TH; a.tiles_n = (N + a.TN - 1) / a.TN;
  HK_REQUIRE((long long)a.tiles_w * a.tiles_h * a.tiles_n < (1ll << 31), HK_ERR_UNSUPPORTED, "conv3x3: grid too large");
  CUtensorMap tmX, tmW;
  int r;
  if ((r = make_act_map(&tmX, x, N, Hin, Win, Cin, a.TW, a.TH, a.TN, stride))) return r;
  const int BN = Cout <= 64 ? 64 : 128;   // 64 accumulator registers per thread at most
  {
    uint64_t dims[3] = {(uint64_t)Cin, (uint64_t)Cout, 9};
    uint64_t strides[2] = {(uint64_t)Cin * 4, (uint64_t)Cin * Cout * 4};
    uint32_t box[3] = {32, (uint32_t)BN, 1};
    if ((r = make_tmap(&tmW, wp, 3, dims, strides, box))) return r;
  }
  if (BN == 64) return launch_conv<64>(tmX, tmW, a, stream);
  return launch_conv<128>(tmX, tmW, a, stream);
}

// ------------------------------------------------------------------------------------------------
// weight gradient: one CTA accumulates dWp[tap][ci0 : ci0 + CI][co0 : co0 + CO] for ALL 9 taps over its share of the
// pixels (split-K across CTAs, fp32 atomics at the end).  A stage covers a 64-pixel tile (TW x TH x TN, a template
// parameter: the fragment addresses and the k-step of every tap are compile-time).  The GEMM is dW^T: M = ci, N = co.
//   A = X (M = 64 ci, k = pixel), in registers.  TMA lands the halo patch, (TH+2) x (TW+2) x TN pixels, as two
//       [pixels][32 ci] boxes (128B-swizzled, zero fill = the conv padding).  Each consumer thread loads its m64k8
//       fragment straight from there: the kw shift of a tap is a row offset, so X is never transposed or copied.
//   B = dY^T (N = 64 co, k = pixel), K-major: the producer warpgroup transposes the two [64 px][32 co] dY boxes once
//       per stage into [co][pixel] (two k-chunks of [64 co][32 px]), one box and k-chunk per warp, and sums the bias
//       gradient on the way.
//   Consumers: warpgroups 1..3, one per kernel column kw.  Warpgroup kw walks the halo rows; the fragment of halo row
//       y (one 8-pixel segment) is the A operand of output row y - kh for each kh with 0 <= y - kh < TH, so it is loaded
//       once and feeds up to three m64n64k8 wgmmas into acc[kh] (3 x 32 fp32 registers per thread): 24 wgmmas per stage
//       and warpgroup, one commit group per fragment.  Two fragment buffers keep two groups in flight: fragment i + 1 is
//       loaded and issued while group i runs, and wgmma_wait<1> then retires group i, whose buffer takes fragment i + 2.
//       The swizzle phase of a fragment row depends on y, the segment, kw and the lane's column; the loads reach at most
//       two threads per bank (8 ci in two 16-byte chunks x 4 consecutive halo rows).
//   Registers: setmaxnreg moves registers from the producer (56) to the consumers (152; 128 x 56 + 3 x 128 x 152 =
//       65536, the whole register file).  ptxas allocates code after setmaxnreg against the new limit, but decides
//       whether wgmmas may stay in flight against the 128 of the 512-thread launch bound: 96 accumulators, two
//       fragments and the addressing just fit (R0..R127), and one more live register (a spin counter in the consumers'
//       full-barrier wait) makes it serialise every wgmma (advisory C7512).  So the consumers wait unguarded, and the
//       producer carries the watchdog: it cannot refill a slot the consumers never released, and at the end it waits
//       guarded on the full phases of the last stages itself.
//   Pipeline: three stage slots {halo boxes, dY^T, raw dY}.  Raw dY of stage k + 3 is requested as soon as stage k's
//       has been transposed; the halo boxes as soon as the three consumer warpgroups release the slot, which each does
//       once the group of the slot's last fragment has retired, one fragment into the next stage (the fragment buffers
//       alternate across stages: a stage has an even number of fragments).  The tile origin advances incrementally (no
//       division inside the loop).
// ------------------------------------------------------------------------------------------------
struct WgradArgs {
  float* dWp;  // [9][Cin][Cout], pre-zeroed
  float* db;   // [Cout], pre-zeroed, or null
  int N, H, W, Cin, Cout;
  int TW, TH, TN, tiles_w, tiles_h, tiles_n;
  int total_tiles, per;   // pixel tiles, and tiles per split-K CTA (blockIdx.y)
};

constexpr int WG_THREADS = 4 * 128;                // the producer warpgroup, then one consumer warpgroup per kernel column
constexpr int WG_PRODUCER_REGS = 56, WG_CONSUMER_REGS = 152;   // setmaxnreg budgets
static_assert(128 * WG_PRODUCER_REGS + 3 * 128 * WG_CONSUMER_REGS <= 65536, "wgrad register budget");
constexpr int WG_STAGES = 3;                       // stage slots
constexpr int WG_KP = 64;                          // pixels per stage
constexpr int WG_RAW_ROWS = 120;                   // (TH + 2) * (TW + 2) * TN: halo box rows (TW >= 8)
constexpr int WG_RAW_BYTES = WG_RAW_ROWS * 128;    // one 32-ci halo box (15 KB, whole swizzle atoms)

constexpr int WG_CI = 64, WG_CO = 64;             // CTA tile
constexpr int WG_X_BYTES = (WG_CI / 32) * WG_RAW_BYTES;
constexpr int WG_DY_BYTES = (WG_CO / 32) * WG_KP * 128;                   // raw dY boxes, and dY^T
constexpr int WG_STAGE_BYTES = WG_X_BYTES + 2 * WG_DY_BYTES;              // {halo boxes, dY^T, raw dY}
constexpr int WG_SMEM = WG_STAGES * WG_STAGE_BYTES + 1024 + 256;          // 186 KB + alignment + barriers
static_assert(WG_SMEM <= 227 * 1024, "wgrad shared memory");

// tile origin (w0, h0, n0) of pixel tile t, advanced one tile at a time
template <int TW, int TH, int TN>
struct WgradTile {
  int w0, h0, n0;
  __device__ __forceinline__ WgradTile(int t, const WgradArgs& a) {
    w0 = t % a.tiles_w * TW; t /= a.tiles_w;
    h0 = t % a.tiles_h * TH;
    n0 = t / a.tiles_h * TN;
  }
  __device__ __forceinline__ void next(const WgradArgs& a) {
    if ((w0 += TW) < a.W) return;
    w0 = 0;
    if ((h0 += TH) < a.H) return;
    h0 = 0;
    n0 += TN;
  }
};

template <int TW, int TH, int TN>
__global__ void __launch_bounds__(WG_THREADS, 1)
conv3x3_wgrad_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX, WgradArgs a) {
  static_assert(TW * TH * TN == WG_KP && TW % 8 == 0, "64-pixel tile of whole 8-pixel rows");
  static_assert((TH + 2) * (TW + 2) * TN <= WG_RAW_ROWS, "halo patch too large");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + WG_STAGES * WG_STAGE_BYTES);
  uint64_t* empty = full + WG_STAGES;
  uint64_t* dy_full = empty + WG_STAGES;
  const uint32_t stage0 = smem_u32(smem);

  const int warp = threadIdx.x >> 5;
  const int n_ci_tiles = (a.Cin + WG_CI - 1) / WG_CI;
  const int ci_t = blockIdx.x % n_ci_tiles, co_t = blockIdx.x / n_ci_tiles;
  const int co0 = co_t * WG_CO, ci0 = ci_t * WG_CI;
  const long long t_begin = (long long)a.per * blockIdx.y;   // < total_tiles < 2^31 for every launched CTA
  const int nk = (int)min((long long)a.per, (long long)a.total_tiles - t_begin);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmDY);
    tma_prefetch_desc(&tmX);
    for (int s = 0; s < WG_STAGES; ++s) {
      mbar_init(&full[s], 2);       // the halo TMA's expect_tx arrival + the producer's once dY^T is written
      mbar_init(&empty[s], 3);      // one arrival per consumer warpgroup
      mbar_init(&dy_full[s], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (nk <= 0) return;

  if (warp < 4) {
    regs_dealloc<WG_PRODUCER_REGS>();
    // warp w transposes k-chunk c = w / 2 (pixels 32 c .. 32 c + 31) of raw dY box j = w % 2: its lane writes row
    // co = 32 j + lane of dY^T (column lane of the box) and sums that part of co's bias
    const int lane = threadIdx.x & 31, j = warp & 1, c = warp >> 1;
    constexpr uint32_t x_tx = (WG_CI / 32) * (TH + 2) * (TW + 2) * TN * 128;
    WgradTile<TW, TH, TN> x_tile((int)t_begin, a), dy_tile = x_tile;   // only thread 0 issues TMAs
    if (threadIdx.x == 0)
      for (int u = 0; u < WG_STAGES && u < nk; ++u) {
        uint8_t* dy = smem + u * WG_STAGE_BYTES + WG_X_BYTES + WG_DY_BYTES;
        mbar_expect_tx(&dy_full[u], WG_DY_BYTES);
#pragma unroll
        for (int b = 0; b < WG_CO / 32; ++b)
          tma_load_4d(dy + b * (WG_KP * 128), &tmDY, &dy_full[u], co0 + b * 32, dy_tile.w0, dy_tile.h0, dy_tile.n0);
        dy_tile.next(a);
      }
    float bsum = 0.f;
    int s = 0;
    uint32_t ph = 0;
    for (int k = 0; k < nk; ++k) {
      uint8_t* st = smem + s * WG_STAGE_BYTES;
      mbar_wait(&empty[s], ph ^ 1);
      if (threadIdx.x == 0) {
        mbar_expect_tx(&full[s], x_tx);
#pragma unroll
        for (int b = 0; b < WG_CI / 32; ++b)
          tma_load_4d(st + b * WG_RAW_BYTES, &tmX, &full[s], ci0 + b * 32, x_tile.w0 - 1, x_tile.h0 - 1, x_tile.n0);
        x_tile.next(a);
      }
      mbar_wait(&dy_full[s], ph);
      const uint32_t dyt = smem_u32(st + WG_X_BYTES), dy = dyt + WG_DY_BYTES;
#pragma unroll
      for (int k4 = 0; k4 < 8; ++k4) {             // pixels 32 c + 4 k4 .. 32 c + 4 k4 + 3
        uint32_t v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          v[i] = ld_shared_u32(dy + j * (WG_KP * 128) + sw128_off(32 * c + 4 * k4 + i, lane));
          bsum += __uint_as_float(v[i]);
        }
        st_shared_v4(dyt + c * (WG_CO * 128) + sw128_off(32 * j + lane, 4 * k4), v[0], v[1], v[2], v[3]);
      }
      fence_proxy_async();
      named_bar(1, 128);                            // dY^T is complete and raw dY slot s is free
      if (threadIdx.x == 0) {
        if (k + WG_STAGES < nk) {
          mbar_expect_tx(&dy_full[s], WG_DY_BYTES);
#pragma unroll
          for (int b = 0; b < WG_CO / 32; ++b)
            tma_load_4d(st + WG_X_BYTES + WG_DY_BYTES + b * (WG_KP * 128), &tmDY, &dy_full[s], co0 + b * 32, dy_tile.w0,
                        dy_tile.h0, dy_tile.n0);
          dy_tile.next(a);
        }
        mbar_arrive(&full[s]);
      }
      if (++s == WG_STAGES) { s = 0; ph ^= 1; }
    }
    // the watchdog for the consumers' unguarded full waits: a stage before the last WG_STAGES was released by them, so
    // its full phase completed; the last ones are checked here
    for (int kk = max(nk - WG_STAGES, 0); kk < nk; ++kk) mbar_wait(&full[kk % WG_STAGES], (kk / WG_STAGES) & 1);
    // bias: added once per co and k-chunk, by the ci-tile-0 CTAs
    if (a.db && ci_t == 0 && co0 + 32 * j + lane < a.Cout) atomicAdd(a.db + co0 + 32 * j + lane, bsum);
  } else {
    regs_alloc<WG_CONSUMER_REGS>();
    const int kw = (warp >> 2) - 1, t = threadIdx.x & 127, wl = t >> 5, lane = t & 31, g = lane >> 2, q = lane & 3;
    // this thread's A rows: ci 16 wl + g (+8) = column cib (+8) of halo box wl / 2.  Its k columns q (+4) of a fragment
    // whose 8 pixels start at halo row R read halo rows R + kw + q (+4).  In a SWIZZLE_128B box the 16-byte chunk of a
    // row is XOR-ed with bits 7..9 of the row's address, which is computed per fragment: a table of phases would cost
    // the registers the wgmma pipeline needs.  cq: chunk and word of ci cib in an unswizzled row.  cib / 4 is 0, 1, 4
    // or 5, so ci cib + 8 is chunk ^ 2 (address ^ 32).
    const int cib = 16 * (wl & 1) + g;
    const uint32_t cq = (uint32_t)(((cib >> 2) << 4) | ((cib & 3) << 2));
    const uint32_t xrow = (uint32_t)((wl >> 1) * WG_RAW_BYTES + (kw + q) * 128);
    float acc[3][32];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int e = 0; e < 32; ++e) acc[j][e] = 0.f;
    uint32_t f[2][4];   // fragment i of a stage goes to f[i % 2]
    constexpr int SEG = TW / 8, NF = TN * (TH + 2) * SEG;   // 8-pixel halo row segments per stage
    static_assert(NF % 2 == 0, "the fragment buffers alternate across stages");
    int s = 0, s_prev = 0;
    uint32_t ph = 0;
    for (int k = 0; k < nk; ++k) {
      mbar_wait_unguarded(&full[s], ph);   // the producer's guarded waits trap if this phase never completes
      const uint32_t xb = stage0 + s * WG_STAGE_BYTES, xa = xb + xrow;
      const uint64_t bdesc = make_sdesc(xb + WG_X_BYTES);
#pragma unroll
      for (int i = 0; i < NF; ++i) {
        const int n = i / ((TH + 2) * SEG), y = i / SEG % (TH + 2), js = i % SEG;
        const int R = (n * (TH + 2) + y) * (TW + 2) + 8 * js;
        const uint32_t r0 = xa + R * 128, r4 = xa + (R + 4) * 128;
        const uint32_t p0 = r0 + (((r0 >> 3) & 0x70) ^ cq), p4 = r4 + (((r4 >> 3) & 0x70) ^ cq);
        uint32_t (&fi)[4] = f[i & 1];   // its previous fragment's group retired at the last wgmma_wait<1>
        fi[0] = ld_shared_u32(p0);
        fi[1] = ld_shared_u32(p0 ^ 32);
        fi[2] = ld_shared_u32(p4);
        fi[3] = ld_shared_u32(p4 ^ 32);
        wgmma_fence();
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
          const int h = y - kh;
          if (h < 0 || h >= TH) continue;
          const int ks = ((n * TH + h) * TW + 8 * js) / 8;   // k-step of output pixels (n, h, 8 js .. 8 js + 7)
          wgmma_tf32(acc[kh], fi, bdesc + (uint32_t)(((ks >> 2) * (WG_CO * 128) + (ks & 3) * 32) >> 4));
        }
        wgmma_commit();
        wgmma_wait<1>();      // retires the previous fragment's group: its buffer takes the next fragment
#pragma unroll
        for (int j = 0; j < 3; ++j) wgmma_keep(acc[j]);
        if (i == 0 && k > 0 && t == 0) mbar_arrive(&empty[s_prev]);   // the previous stage's last group has retired
      }
      s_prev = s;
      if (++s == WG_STAGES) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 3; ++j) wgmma_keep(acc[j]);
    // accumulator element 4 i + e: ci row 16 wl + g + 8 (e >> 1), co columns 8 i + 2 q (+1), adjacent in dWp
#pragma unroll
    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
      for (int e = 0; e < 32; e += 2) {
        const int ci = ci0 + 16 * wl + g + 8 * ((e >> 1) & 1);
        const int co = co0 + 8 * (e >> 2) + 2 * q;
        if (ci < a.Cin && co < a.Cout)
          atomicAdd(reinterpret_cast<float2*>(a.dWp + ((size_t)(3 * kh + kw) * a.Cin + ci) * a.Cout + co),
                    make_float2(acc[kh][e], acc[kh][e + 1]));
      }
  }
}

// pixel tile for wgrad: TW in {8,16} (a fragment is 8 pixels of one tile row), TW*TH*TN = 64, TH*TW % 8 == 0.
// Returns one of the three tiles launch_wgrad instantiates: (16, 4, 1), (8, 8, 1), (8, 4, 2).
static bool pick_wgrad_tile(int W, int H, int* TW, int* TH, int* TN) {
  int tw = 0;
  for (int c : {16, 8}) if (W % c == 0) { tw = c; break; }
  if (!tw) tw = W <= 8 ? 8 : 16;   // over-wide tile: out-of-range columns are TMA zero fill
  int th = 1;
  while (th * 2 * tw <= 64 && H % (th * 2) == 0) th *= 2;
  int tn = 64 / (tw * th);
  if ((th * tw) % 8 != 0 || (th + 2) * (tw + 2) * tn > WG_RAW_ROWS) {   // fall back to one image per tile, partial tiles in H allowed
    th = 64 / tw;
    tn = 1;
  }
  *TW = tw; *TH = th; *TN = tn;
  return true;
}

template <int TW, int TH, int TN>
static int launch_wgrad_tile(const CUtensorMap& tmDY, const CUtensorMap& tmX, const WgradArgs& a, dim3 grid,
                             cudaStream_t stream) {
  int r;
  if ((r = allow_dynamic_smem<conv3x3_wgrad_kernel<TW, TH, TN>>(WG_SMEM, "wgrad"))) return r;
  conv3x3_wgrad_kernel<TW, TH, TN><<<grid, WG_THREADS, WG_SMEM, stream>>>(tmDY, tmX, a);
  HK_LAUNCH_CHECK("conv3x3_wgrad_kernel");
  return 0;
}

static int launch_wgrad(const float* x, const float* dy, WgradArgs a, cudaStream_t stream) {
  const long long out_tiles = (long long)((a.Cout + WG_CO - 1) / WG_CO) * ((a.Cin + WG_CI - 1) / WG_CI);
  const long long total_tiles = (long long)a.tiles_w * a.tiles_h * a.tiles_n;
  HK_REQUIRE(total_tiles < (1ll << 31), HK_ERR_UNSUPPORTED, "conv3x3_wgrad: too many pixel tiles");
  // split-K factor.  The kernel runs one CTA per SM (its 186 KB of shared memory allow no second, and its 512 threads
  // hold the whole register file), so the grid executes in whole waves of `sms` CTAs: pick the split that fills
  // 1..3 waves best (ties -> fewer waves: fewer partial sums to add).
  const int sms = num_sms();
  long long ks = 1;
  {
    double best = -1.0;
    for (int w = 1; w <= 3; ++w) {
      long long k = (long long)sms * w / out_tiles;
      if (k < 1) k = 1;
      if (k > total_tiles) k = total_tiles;
      const long long ctas = k * out_tiles;
      const long long waves = (ctas + sms - 1) / sms;
      const double fill = (double)ctas / (double)(waves * sms);
      if (fill > best + 1e-9) { best = fill; ks = k; }
    }
  }
  if (ks > total_tiles) ks = total_tiles;
  if (ks < 1) ks = 1;
  if (ks > 65535) ks = 65535;
  a.total_tiles = (int)total_tiles;
  a.per = (int)((total_tiles + ks - 1) / ks);
  const dim3 grid((unsigned)out_tiles, (unsigned)((total_tiles + a.per - 1) / a.per));   // every CTA has tiles
  CUtensorMap tmDY, tmX;
  int r;
  if ((r = make_act_map(&tmDY, dy, a.N, a.H, a.W, a.Cout, a.TW, a.TH, a.TN))) return r;
  if ((r = make_act_map(&tmX, x, a.N, a.H, a.W, a.Cin, a.TW + 2, a.TH + 2, a.TN))) return r;
  if (a.TW == 16 && a.TH == 4 && a.TN == 1) return launch_wgrad_tile<16, 4, 1>(tmDY, tmX, a, grid, stream);
  if (a.TW == 8 && a.TH == 8 && a.TN == 1) return launch_wgrad_tile<8, 8, 1>(tmDY, tmX, a, grid, stream);
  if (a.TW == 8 && a.TH == 4 && a.TN == 2) return launch_wgrad_tile<8, 4, 2>(tmDY, tmX, a, grid, stream);
  return set_error(HK_ERR_UNSUPPORTED, "conv3x3_wgrad: pixel tile %dx%dx%d has no kernel", a.TW, a.TH, a.TN);
}

static int conv3x3_wgrad_1x(const float* x, const float* dy, float* dwp, float* db, int N, int H, int W, int Cin, int Cout,
                            cudaStream_t stream, bool zero_dw, bool zero_db);

int conv3x3_wgrad(const float* x, const float* dy, float* dwp, float* db, int N, int H, int W, int Cin, int Cout,
                  cudaStream_t stream, bool zero_db = true) {
  if (!precise()) return conv3x3_wgrad_1x(x, dy, dwp, db, N, H, W, Cin, Cout, stream, true, zero_db);
  // 3xTF32: dW = dYh^T Xh + dYh^T Xl + dYl^T Xh accumulated by the kernel's own atomics; db = sum(dYh) + sum(dYl)
  HK_REQUIRE(x && dy && dwp, HK_ERR_ARG, "conv3x3_wgrad: null pointer");
  const size_t nx = (size_t)N * H * W * Cin, ny = (size_t)N * H * W * Cout;
  Scratch sx(2 * nx * sizeof(float), stream), sy(2 * ny * sizeof(float), stream);
  HK_REQUIRE(sx.p && sy.p, HK_ERR_DRIVER, "conv3x3_wgrad (precise): cudaMallocAsync of the operand halves failed");
  float *xh = sx.f(), *xl = xh + nx, *yh = sy.f(), *yl = yh + ny;
  int r;
  if ((r = tf32_split(x, xh, xl, nx, stream))) return r;
  if ((r = tf32_split(dy, yh, yl, ny, stream))) return r;
  if ((r = conv3x3_wgrad_1x(xh, yh, dwp, db, N, H, W, Cin, Cout, stream, true, zero_db))) return r;
  if ((r = conv3x3_wgrad_1x(xl, yh, dwp, nullptr, N, H, W, Cin, Cout, stream, false, false))) return r;
  return conv3x3_wgrad_1x(xh, yl, dwp, db, N, H, W, Cin, Cout, stream, false, false);
}

static int conv3x3_wgrad_1x(const float* x, const float* dy, float* dwp, float* db, int N, int H, int W, int Cin, int Cout,
                            cudaStream_t stream, bool zero_dw, bool zero_db) {
  HK_REQUIRE(x && dy && dwp, HK_ERR_ARG, "conv3x3_wgrad: null pointer");
  HK_REQUIRE(Cin % 32 == 0 && Cout % 32 == 0, HK_ERR_UNSUPPORTED, "conv3x3_wgrad: Cin=%d Cout=%d unsupported", Cin, Cout);
  WgradArgs a = {};
  a.dWp = dwp; a.db = db; a.N = N; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout;
  pick_wgrad_tile(W, H, &a.TW, &a.TH, &a.TN);
  HK_REQUIRE((a.TH + 2) * (a.TW + 2) * a.TN <= WG_RAW_ROWS, HK_ERR_UNSUPPORTED,
             "conv3x3_wgrad: halo patch too large");
  a.tiles_w = (W + a.TW - 1) / a.TW; a.tiles_h = (H + a.TH - 1) / a.TH; a.tiles_n = (N + a.TN - 1) / a.TN;
  cudaError_t e = cudaSuccess;
  if (zero_dw) {
    e = cudaMemsetAsync(dwp, 0, (size_t)9 * Cout * Cin * sizeof(float), stream);
    if (e != cudaSuccess) return set_error((int)e, "cudaMemsetAsync(dWp): %s", cudaGetErrorString(e));
  }
  if (db && zero_db) {
    e = cudaMemsetAsync(db, 0, (size_t)Cout * sizeof(float), stream);
    if (e != cudaSuccess) return set_error((int)e, "cudaMemsetAsync(db): %s", cudaGetErrorString(e));
  }
  return launch_wgrad(x, dy, a, stream);
}

// ------------------------------------------------------------------------------------------------
// first layer (Cin = 3; vgg.py:61 in_channels=3): im2col to X27 + one wgmma GEMM (see hk_conv3x3_first_fwd)
// ------------------------------------------------------------------------------------------------
// first-layer weight gradient on the tensor cores: materialise the 3x3x3 patches as X27 [pix][32]
// (27 taps, column 27 = 1.0 so that the GEMM's column 27 is the bias gradient, columns 28..31 = 0) and run
// dW^T-partials[s] = dY[pix-range s]^T . X27[pix-range s]  as a batched (split-K) MN-major wgmma GEMM.
__global__ void im2col_first_kernel(const float* __restrict__ x, float* __restrict__ x27, int N, int H, int W, int round) {
  const long long total = (long long)N * H * W;
  for (long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x; pix < total;
       pix += (long long)gridDim.x * blockDim.x) {
    const int wq = (int)(pix % W), hq = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
    float v[32];
#pragma unroll
    for (int ci = 0; ci < 3; ++ci)
#pragma unroll
      for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int hh = hq + kh - 1, ww = wq + kw - 1;
          float t = (hh >= 0 && hh < H && ww >= 0 && ww < W) ? __ldg(x + (((size_t)n * 3 + ci) * H + hh) * W + ww) : 0.f;
          v[ci * 9 + kh * 3 + kw] = round ? tf32_round(t) : t;
        }
    v[27] = 1.f; v[28] = v[29] = v[30] = v[31] = 0.f;
    float4* dst = reinterpret_cast<float4*>(x27 + (size_t)pix * 32);
#pragma unroll
    for (int j = 0; j < 8; ++j) dst[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
  }
}
// w27[co][0..26] = tf32(w[co][ci][kh][kw]), w27[co][27] = bias[co] (x27 column 27 is 1.0), rest 0
__global__ void pack_first_weights_kernel(const float* __restrict__ w, const float* __restrict__ bias,
                                          float* __restrict__ w27, int Cout, int round) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Cout * 32) return;
  const int co = i / 32, r = i % 32;
  const float t = r < 27 ? w[co * 27 + r] : (r == 27 && bias ? bias[co] : 0.f);
  w27[i] = round ? tf32_round(t) : t;
}

// tf32(x[n][ci][h + kh - 1][w + kw - 1]) for X27 column j = 9 ci + 3 kh + kw < 27 (zero padding), 1.0 for j = 27, 0 after:
// the row of X27 that im2col_first_kernel writes, rebuilt where it is consumed.
__device__ __forceinline__ float x27_value(const float* __restrict__ x, int n, int hq, int wq, int j, int H, int W) {
  if (j >= 27) return j == 27 ? 1.f : 0.f;
  const int ci = j / 9, hh = hq + (j % 9) / 3 - 1, ww = wq + j % 3 - 1;
  return (hh >= 0 && hh < H && ww >= 0 && ww < W) ? tf32_round(__ldg(x + (((size_t)n * 3 + ci) * H + hh) * W + ww)) : 0.f;
}

// First-layer forward without X27 in memory: y = tf32(relu(X27 . W27^T)) for Cout = 64.  One warpgroup per 128 pixels:
// each thread writes its pixel's X27 row and two W27 rows into 128B-swizzled K-major tiles, then the warpgroup issues
// the same four m64n64k8 k-steps per 64 rows as the GEMM of hk_conv3x3_first_fwd, so y is bit-identical to it.
constexpr int FIRST_FWD_PIX = 128;
constexpr int FIRST_FWD_SMEM = 1024 + FIRST_FWD_PIX * 128 + 64 * 128;
__global__ void __launch_bounds__(128) first_fwd_direct_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                               const float* __restrict__ bias, float* __restrict__ y,
                                                               int N, int H, int W) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sA = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sB = sA + FIRST_FWD_PIX * 128;
  const int t = threadIdx.x;
  const long long P = (long long)N * H * W, p0 = (long long)blockIdx.x * FIRST_FWD_PIX;
  {
    const long long p = p0 + t;
    float v[32];
    if (p < P) {
      const int wq = (int)(p % W), hq = (int)((p / W) % H), n = (int)(p / ((long long)W * H));
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = x27_value(x, n, hq, wq, j, H, W);
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 32; j += 4)
      *reinterpret_cast<float4*>(sA + sw128_off(t, j)) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
    // W27 (pack_first_weights_kernel's layout): thread t fills columns 16 (t & 1) .. + 15 of row t / 2
    const int co = t >> 1, c0 = (t & 1) * 16;
#pragma unroll
    for (int j = 0; j < 16; j += 4) {
      float4 q;
      float* qq = reinterpret_cast<float*>(&q);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = c0 + j + e;
        qq[e] = tf32_round(r < 27 ? __ldg(w + co * 27 + r) : (r == 27 && bias ? __ldg(bias + co) : 0.f));
      }
      *reinterpret_cast<float4*>(sB + sw128_off(co, c0 + j)) = q;
    }
  }
  fence_proxy_async();
  __syncthreads();
  const uint64_t b_base = make_sdesc(smem_u32(sB));
  float acc[2][32];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[m][i] = 0.f;
  wgmma_fence();
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    const uint64_t a_base = make_sdesc(smem_u32(sA + m * 64 * 128));
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_tf32(acc[m], a_base + ks * 2, b_base + ks * 2, 1);
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_keep(acc[0]);
  wgmma_keep(acc[1]);
  // fragment (row 16 warp + lane / 4 (+8), columns 8 i + 2 (lane % 4) (+1)): four lanes fill one 32-byte sector
  const int warp = t >> 5, lane = t & 31;
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long p = p0 + m * 64 + warp * 16 + (lane >> 2) + 8 * h;
      if (p >= P) continue;
      float* dst = y + p * 64 + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<float2*>(dst + 8 * i) =
            make_float2(tf32_round(fmaxf(acc[m][4 * i + 2 * h], 0.f)), tf32_round(fmaxf(acc[m][4 * i + 2 * h + 1], 0.f)));
    }
}

// First-layer weight and bias gradient without X27 in memory, Cout = 64: part[cta] = dY^T . X27 over the pixels of the
// CTA, on register-A m64n32k8 wgmma.  Each warpgroup takes 32-pixel blocks in turn: A = dY^T read straight from the NHWC
// dY into the fragment layout (four lanes read one 32-byte sector), B = the block's X27 rebuilt from the image as a
// [32 column][32 pixel] K-major tile.  The two warpgroups' sums meet in shared memory; sum_splits reduces the CTAs.
constexpr int FIRST_WG_THREADS = 256;
constexpr int FIRST_WG_SMEM = 1024 + 64 * 33 * 4;     // two 4 KB B tiles, then the [64][33] reduction tile
__global__ void __launch_bounds__(FIRST_WG_THREADS, 2) first_wgrad_direct_kernel(const float* __restrict__ x,
                                                                              const float* __restrict__ dy,
                                                                              float* __restrict__ part, int N, int H, int W) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
  uint8_t* sB = smem + wg * 32 * 128;
  const int P = N * H * W, nblk = (P + 31) / 32;     // P < 2^31 (checked by the entry)
  const uint64_t b_base = make_sdesc(smem_u32(sB));
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  const int co = warp * 16 + (lane >> 2);
  for (int blk = blockIdx.x * 2 + wg; blk < nblk; blk += gridDim.x * 2) {
    const int pb = blk * 32;
    uint32_t a[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int p = pb + 8 * ks + (lane & 3) + 4 * (e >> 1);
        a[ks][e] = p < P ? __float_as_uint(__ldg(dy + (size_t)p * 64 + co + 8 * (e & 1))) : 0u;
      }
    float v[8];
    {
      const int p = pb + lane;
      if (p < P) {
        const int wq = p % W, hq = (p / W) % H, n = p / (W * H);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) v[jj] = x27_value(x, n, hq, wq, warp * 8 + jj, H, W);
      } else {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) v[jj] = 0.f;
      }
    }
    named_bar(1 + wg, 128);     // the previous block's wgmma has completed in every warp: sB may be overwritten
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) *reinterpret_cast<float*>(sB + sw128_off(warp * 8 + jj, lane)) = v[jj];
    fence_proxy_async();
    named_bar(1 + wg, 128);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_tf32(acc, a[ks], b_base + ks * 2);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_keep(acc);
  }
  __syncthreads();
  float* red = reinterpret_cast<float*>(smem);     // [64][33], over the (now idle) B tiles
  if (wg == 1) {
#pragma unroll
    for (int i = 0; i < 16; ++i) red[(co + 8 * ((i >> 1) & 1)) * 33 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1)] = acc[i];
  }
  __syncthreads();
  if (wg == 0) {
    float* dst = part + (size_t)blockIdx.x * 64 * 32;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int r = co + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      dst[r * 32 + c] = acc[i] + red[r * 33 + c];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// MaxPool2d(2,2) (vgg.py:59) on NHWC; optional NCHW output for the last pool (feeds the pooling head)
// ------------------------------------------------------------------------------------------------
__global__ void maxpool2x2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int H, int W, int C,
                                      int out_nchw) {
  const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
  const size_t total = (size_t)N * Ho * Wo * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    size_t p = i / C4;
    const int wo = p % Wo; p /= Wo;
    const int ho = p % Ho;
    const int n = p / Ho;
    const float4* base = reinterpret_cast<const float4*>(x + (((size_t)n * H + 2 * ho) * W + 2 * wo) * C) + c4;
    const float4 a = base[0], b = base[C4], c = base[(size_t)W * C4], d = base[(size_t)W * C4 + C4];
    float4 m;
    m.x = fmaxf(fmaxf(a.x, b.x), fmaxf(c.x, d.x));
    m.y = fmaxf(fmaxf(a.y, b.y), fmaxf(c.y, d.y));
    m.z = fmaxf(fmaxf(a.z, b.z), fmaxf(c.z, d.z));
    m.w = fmaxf(fmaxf(a.w, b.w), fmaxf(c.w, d.w));
    if (!out_nchw) {
      reinterpret_cast<float4*>(y + (((size_t)n * Ho + ho) * Wo + wo) * C)[c4] = m;
    } else {
      const size_t hw = (size_t)Ho * Wo, o = ((size_t)n * C + c4 * 4) * hw + (size_t)ho * Wo + wo;
      y[o] = m.x; y[o + hw] = m.y; y[o + 2 * hw] = m.z; y[o + 3 * hw] = m.w;
    }
  }
}

// backward: dx[window] = dy routed to the first max in scan order (PyTorch max_pool2d_backward), then multiplied by
// (x > 0): x is the ReLU output feeding the pool, so this also applies the preceding ReLU's backward.
__global__ void maxpool2x2_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                      float* __restrict__ dx, int N, int H, int W, int C, int dy_nchw) {
  const int Ho = H / 2, Wo = W / 2;
  const size_t total = (size_t)N * Ho * Wo * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = i % C;
    size_t p = i / C;
    const int wo = p % Wo; p /= Wo;
    const int ho = p % Ho;
    const int n = p / Ho;
    const size_t b00 = (((size_t)n * H + 2 * ho) * W + 2 * wo) * C + c;
    const size_t b01 = b00 + C, b10 = b00 + (size_t)W * C, b11 = b10 + C;
    const float v00 = x[b00], v01 = x[b01], v10 = x[b10], v11 = x[b11];
    const float g = dy_nchw ? dy[((size_t)n * C + c) * Ho * Wo + (size_t)ho * Wo + wo] : dy[i];
    int arg = 0;
    float m = v00;
    if (v01 > m) { m = v01; arg = 1; }
    if (v10 > m) { m = v10; arg = 2; }
    if (v11 > m) { m = v11; arg = 3; }
    const float gm = m > 0.f ? g : 0.f;
    dx[b00] = arg == 0 ? gm : 0.f;
    dx[b01] = arg == 1 ? gm : 0.f;
    dx[b10] = arg == 2 ? gm : 0.f;
    dx[b11] = arg == 3 ? gm : 0.f;
  }
}

// Training variants: the forward also records, per pooled element, ONE byte — bits 0-1 = window position of the first
// maximum in scan order (PyTorch routing), bit 2 = (max > 0), i.e. the mask of the ReLU that precedes the pool — and the
// backward routes dy from that byte alone: it no longer re-reads the four pre-pool activations (1/16 of the bytes).
__global__ void maxpool2x2_fwd_idx_kernel(const float* __restrict__ x, float* __restrict__ y, unsigned char* __restrict__ code,
                                          int N, int H, int W, int C, int out_nchw) {
  const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
  const size_t total = (size_t)N * Ho * Wo * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    size_t p = i / C4;
    const int wo = p % Wo; p /= Wo;
    const int ho = p % Ho;
    const int n = p / Ho;
    const float4* base = reinterpret_cast<const float4*>(x + (((size_t)n * H + 2 * ho) * W + 2 * wo) * C) + c4;
    const float4 v0 = base[0], v1 = base[C4], v2 = base[(size_t)W * C4], v3 = base[(size_t)W * C4 + C4];
    float4 m = v0;
    uchar4 a = make_uchar4(0, 0, 0, 0);
#define HK_POOL_STEP(V, K)                     \
    if (V.x > m.x) { m.x = V.x; a.x = K; }     \
    if (V.y > m.y) { m.y = V.y; a.y = K; }     \
    if (V.z > m.z) { m.z = V.z; a.z = K; }     \
    if (V.w > m.w) { m.w = V.w; a.w = K; }
    HK_POOL_STEP(v1, 1) HK_POOL_STEP(v2, 2) HK_POOL_STEP(v3, 3)
#undef HK_POOL_STEP
    a.x |= m.x > 0.f ? 4 : 0; a.y |= m.y > 0.f ? 4 : 0; a.z |= m.z > 0.f ? 4 : 0; a.w |= m.w > 0.f ? 4 : 0;
    reinterpret_cast<uchar4*>(code)[i] = a;
    if (!out_nchw) {
      reinterpret_cast<float4*>(y + (((size_t)n * Ho + ho) * Wo + wo) * C)[c4] = m;
    } else {
      const size_t hw = (size_t)Ho * Wo, o = ((size_t)n * C + c4 * 4) * hw + (size_t)ho * Wo + wo;
      y[o] = m.x; y[o + hw] = m.y; y[o + 2 * hw] = m.z; y[o + 3 * hw] = m.w;
    }
  }
}
__global__ void maxpool2x2_bwd_idx_kernel(const unsigned char* __restrict__ code, const float* __restrict__ dy,
                                          float* __restrict__ dx, int N, int H, int W, int C, int dy_nchw) {
  const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
  const size_t total = (size_t)N * Ho * Wo * C4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = i % C4;
    size_t p = i / C4;
    const int wo = p % Wo; p /= Wo;
    const int ho = p % Ho;
    const int n = p / Ho;
    const uchar4 a = reinterpret_cast<const uchar4*>(code)[i];
    float4 g;
    if (!dy_nchw) {
      g = reinterpret_cast<const float4*>(dy)[i];
    } else {
      const size_t hw = (size_t)Ho * Wo, o = ((size_t)n * C + c4 * 4) * hw + (size_t)ho * Wo + wo;
      g = make_float4(dy[o], dy[o + hw], dy[o + 2 * hw], dy[o + 3 * hw]);
    }
    g.x = (a.x & 4) ? g.x : 0.f; g.y = (a.y & 4) ? g.y : 0.f; g.z = (a.z & 4) ? g.z : 0.f; g.w = (a.w & 4) ? g.w : 0.f;
    float4* base = reinterpret_cast<float4*>(dx + (((size_t)n * H + 2 * ho) * W + 2 * wo) * C) + c4;
#define HK_POOL_OUT(K) make_float4((a.x & 3) == K ? g.x : 0.f, (a.y & 3) == K ? g.y : 0.f, (a.z & 3) == K ? g.z : 0.f, \
                                   (a.w & 3) == K ? g.w : 0.f)
    base[0] = HK_POOL_OUT(0);
    base[C4] = HK_POOL_OUT(1);
    base[(size_t)W * C4] = HK_POOL_OUT(2);
    base[(size_t)W * C4 + C4] = HK_POOL_OUT(3);
#undef HK_POOL_OUT
  }
}

// db[c] = sum over pixels of dy[pix][c]   (NHWC)
__global__ void bias_grad_kernel(const float* __restrict__ dy, float* __restrict__ db, size_t npix, int C) {
  // block handles a slab of pixels; threads stride over channels (coalesced), atomics at the end
  const int c = threadIdx.x % C;
  const int lanes_per_c = blockDim.x / C > 0 ? blockDim.x / C : 1;
  const int sub = threadIdx.x / C;
  if (sub >= lanes_per_c) return;
  const size_t per = (npix + gridDim.x - 1) / gridDim.x;
  const size_t p0 = blockIdx.x * per, p1 = (p0 + per < npix) ? p0 + per : npix;
  for (int cc = c; cc < C; cc += (blockDim.x < C ? blockDim.x : C)) {
    float s = 0.f;
    for (size_t p = p0 + sub; p < p1; p += lanes_per_c) s += dy[p * C + cc];
    atomicAdd(db + cc, s);
  }
}

}  // namespace hk

using namespace hk;

extern "C" {

int hk_conv3x3_pack_weights(const float* w, float* w_fwd, float* w_dgrad, int Cout, int Cin, void* stream) {
  HK_REQUIRE(w && (w_fwd || w_dgrad), HK_ERR_ARG, "hk_conv3x3_pack_weights: null pointer");
  pack_weights_kernel<<<grid_1d((size_t)Cout * Cin * 9, 256), 256, 0, (cudaStream_t)stream>>>(w, w_fwd, w_dgrad, Cout, Cin,
                                                                                              precise() ? 0 : 1);
  HK_LAUNCH_CHECK("pack_weights_kernel");
  return 0;
}

int hk_conv3x3_fwd(const float* x, const float* w_packed, const float* bias, float* y, int N, int H, int W, int Cin,
                   int Cout, int relu, void* stream) {
  return conv3x3_igemm(x, w_packed, bias, nullptr, y, N, H, W, Cin, Cout, relu, (cudaStream_t)stream);
}

/* relu(conv3x3(x) + bias) followed by MaxPool2d(2,2) in ONE kernel: the full-resolution map is never written.  pooled:
 * [N,H/2,W/2,Cout] (NHWC) or [N,Cout,H/2,W/2] (out_nchw); code (optional): the byte per pooled element hk_maxpool2x2_bwd_idx
 * consumes.  Bit-identical to hk_conv3x3_fwd + hk_maxpool2x2_fwd_idx.  Single-pass TF32 only (HK_ERR_UNSUPPORTED in precise mode). */
int hk_conv3x3_fwd_pool(const float* x, const float* w_packed, const float* bias, float* pooled, unsigned char* code, int N,
                        int H, int W, int Cin, int Cout, int out_nchw, void* stream) {
  HK_REQUIRE(!precise(), HK_ERR_UNSUPPORTED, "hk_conv3x3_fwd_pool: not available in 3xTF32 mode (use conv + pool)");
  HK_REQUIRE(pooled, HK_ERR_ARG, "hk_conv3x3_fwd_pool: null output");
  return conv3x3_igemm_1x(x, w_packed, bias, nullptr, nullptr, nullptr, N, H, W, Cin, Cout, 1, (cudaStream_t)stream, 1,
                          0, pooled, code, out_nchw);
}

int hk_conv3x3_s2_fwd(const float* x, const float* w_packed, const float* bias, float* y, int N, int H, int W, int Cin,
                      int Cout, int relu, void* stream) {
  return conv3x3_igemm(x, w_packed, bias, nullptr, y, N, H, W, Cin, Cout, relu, (cudaStream_t)stream, 2);
}

int hk_conv3x3_dgrad(const float* dy, const float* w_dgrad_packed, const float* relu_mask_act, float* dx, int N, int H,
                     int W, int Cin, int Cout, void* stream) {
  // dgrad is the same implicit GEMM with the roles of Cin/Cout swapped and flipped taps
  return conv3x3_igemm(dy, w_dgrad_packed, nullptr, relu_mask_act, dx, N, H, W, Cout, Cin, 0, (cudaStream_t)stream);
}

int hk_conv3x3_dgrad_unpool(const float* dy, const float* w_dgrad_packed, const unsigned char* code, float* dx_full, int N,
                            int H, int W, int Cin, int Cout, void* stream) {
  HK_REQUIRE(!precise(), HK_ERR_UNSUPPORTED, "hk_conv3x3_dgrad_unpool: not available in 3xTF32 mode");
  HK_REQUIRE(dy && w_dgrad_packed && code && dx_full, HK_ERR_ARG, "hk_conv3x3_dgrad_unpool: null pointer");
  HK_REQUIRE(N > 0 && H > 0 && W > 0, HK_ERR_ARG, "hk_conv3x3_dgrad_unpool: empty map");
  HK_REQUIRE(Cin % 32 == 0 && Cout % 32 == 0, HK_ERR_UNSUPPORTED,
             "hk_conv3x3_dgrad_unpool: Cin=%d Cout=%d must be multiples of 32", Cin, Cout);
  HK_REQUIRE(H % 8 == 0 && W % 8 == 0, HK_ERR_UNSUPPORTED, "hk_conv3x3_dgrad_unpool: %dx%d map is not a multiple of 8x8",
             H, W);
  // the epilogue keeps full-resolution element offsets inside a tile (up to one image apart) as int
  HK_REQUIRE(4ll * H * W * Cin < (1ll << 31), HK_ERR_UNSUPPORTED, "hk_conv3x3_dgrad_unpool: map too large");
  HK_REQUIRE(aligned16(dy) && aligned16(w_dgrad_packed) && aligned16(code) && aligned16(dx_full), HK_ERR_ALIGN,
             "hk_conv3x3_dgrad_unpool: pointer not 16-byte aligned");
  ConvArgs a = {};
  a.Y = dx_full; a.code = const_cast<unsigned char*>(code);
  a.N = N; a.H = H; a.W = W; a.Cin = Cout; a.Cout = Cin; a.stride = 1;
  if (W % 16 == 0) return launch_conv_v2<16, EPI_UNPOOL>(dy, w_dgrad_packed, a, N, H, W, (cudaStream_t)stream);
  return launch_conv_v2<8, EPI_UNPOOL>(dy, w_dgrad_packed, a, N, H, W, (cudaStream_t)stream);
}

size_t hk_conv3x3_dgrad_first_wgrad_workspace_bytes(void) { return (size_t)num_sms() * 64 * 32 * sizeof(float); }

int hk_conv3x3_dgrad_first_wgrad_acc(const float* dy, const float* w_dgrad_packed, const float* relu_mask_act,
                                     const float* x_nchw, float* dw1, float* db1, int N, int H, int W, int Cin, int Cout,
                                     void* workspace, size_t workspace_bytes, int accumulate, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  HK_REQUIRE(!precise(), HK_ERR_UNSUPPORTED, "hk_conv3x3_dgrad_first_wgrad: not available in 3xTF32 mode");
  HK_REQUIRE(dy && w_dgrad_packed && x_nchw && dw1, HK_ERR_ARG, "hk_conv3x3_dgrad_first_wgrad: null pointer");
  HK_REQUIRE(N > 0 && H > 0 && W > 0, HK_ERR_ARG, "hk_conv3x3_dgrad_first_wgrad: empty map");
  HK_REQUIRE(Cin == 64 && Cout == 64, HK_ERR_UNSUPPORTED, "hk_conv3x3_dgrad_first_wgrad: Cin=%d Cout=%d (64 -> 64 only)",
             Cin, Cout);
  HK_REQUIRE(W % 16 == 0 && H % 8 == 0, HK_ERR_UNSUPPORTED,
             "hk_conv3x3_dgrad_first_wgrad: %dx%d map is not tiled by 16x8", H, W);
  HK_REQUIRE(aligned16(dy) && aligned16(w_dgrad_packed) && (!relu_mask_act || aligned16(relu_mask_act)), HK_ERR_ALIGN,
             "hk_conv3x3_dgrad_first_wgrad: pointer not 16-byte aligned");
  HK_REQUIRE(workspace && workspace_bytes >= hk_conv3x3_dgrad_first_wgrad_workspace_bytes(), HK_ERR_WORKSPACE,
             "hk_conv3x3_dgrad_first_wgrad: workspace too small");
  const long long tiles = (long long)(W / 16) * (H / 8) * N;
  HK_REQUIRE(tiles < (1ll << 31), HK_ERR_UNSUPPORTED, "hk_conv3x3_dgrad_first_wgrad: too many tiles");
  float* part = static_cast<float*>(workspace);
  ConvArgs a = {};
  a.mask = relu_mask_act;
  a.N = N; a.H = H; a.W = W; a.Cin = Cout; a.Cout = Cin; a.stride = 1;
  int r = launch_conv_v2<64, true, 16, EPI_FIRST_WGRAD>(dy, w_dgrad_packed, a, N, H, W, stream, FirstWgradArgs{x_nchw, part});
  if (r) return r;
  const int G = tiles < num_sms() ? (int)tiles : num_sms();   // launch_conv_v2's grid: one partial per CTA
  // partial columns 0..26 are dw[co][27]; column 27 (the ones column of X27) is db
  if ((r = sum_splits(part, G, 64 * 32, 64, 27, 32, dw1, 27, nullptr, accumulate, stream))) return r;
  if (!db1) return 0;
  return sum_splits(part + 27, G, 64 * 32, 64, 1, 32, db1, 1, nullptr, accumulate, stream);
}

size_t hk_conv3x3_wgrad_workspace_bytes(int Cin, int Cout) { return (size_t)9 * Cin * Cout * sizeof(float); }

int hk_conv3x3_wgrad_acc(const float* x, const float* dy, float* dw, float* db, int N, int H, int W, int Cin, int Cout,
                         void* workspace, size_t workspace_bytes, int accumulate, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  HK_REQUIRE(workspace && workspace_bytes >= hk_conv3x3_wgrad_workspace_bytes(Cin, Cout), HK_ERR_WORKSPACE,
             "hk_conv3x3_wgrad: workspace too small");
  HK_REQUIRE(dw, HK_ERR_ARG, "hk_conv3x3_wgrad: null dw");
  float* dwp = static_cast<float*>(workspace);
  int r = conv3x3_wgrad(x, dy, dwp, db, N, H, W, Cin, Cout, stream, /*zero_db=*/!accumulate);
  if (r) return r;
  unpack_wgrad_kernel<<<grid_1d((size_t)Cout * Cin * 9, 256), 256, 0, stream>>>(dwp, dw, Cout, Cin, accumulate ? 1 : 0);
  HK_LAUNCH_CHECK("unpack_wgrad_kernel");
  return 0;
}

int hk_conv3x3_wgrad(const float* x, const float* dy, float* dw, float* db, int N, int H, int W, int Cin, int Cout,
                     void* workspace, size_t workspace_bytes, void* stream_) {
  return hk_conv3x3_wgrad_acc(x, dy, dw, db, N, H, W, Cin, Cout, workspace, workspace_bytes, 0, stream_);
}

size_t hk_conv3x3_first_fwd_workspace_bytes(int N, int H, int W, int Cout) {
  return ((size_t)N * H * W * 32 + (size_t)Cout * 32) * sizeof(float);
}

/* y = relu(conv3x3(x) + bias) for the 3-channel input layer: patches are materialised once as X27 [pix][32]
 * (tf32-rounded, column 27 = 1 carries the bias) and the layer is ONE wgmma GEMM  y = relu(X27 . W27^T).
 * workspace = X27 followed by W27; X27 (the first N*H*W*32 floats) is what hk_conv3x3_first_wgrad consumes. */
int hk_conv3x3_first_fwd(const float* x_nchw, const float* w, const float* bias, float* y_nhwc, int N, int H, int W,
                         int Cout, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  HK_REQUIRE(x_nchw && w && y_nhwc, HK_ERR_ARG, "hk_conv3x3_first_fwd: null pointer");
  HK_REQUIRE(Cout % 4 == 0 && Cout <= 256, HK_ERR_UNSUPPORTED, "hk_conv3x3_first_fwd: Cout=%d unsupported", Cout);
  HK_REQUIRE(workspace && workspace_bytes >= hk_conv3x3_first_fwd_workspace_bytes(N, H, W, Cout), HK_ERR_WORKSPACE,
             "hk_conv3x3_first_fwd: workspace too small");
  const long long P = (long long)N * H * W;
  HK_REQUIRE(P < (1ll << 31), HK_ERR_UNSUPPORTED, "hk_conv3x3_first_fwd: too many pixels");
  float* x27 = static_cast<float*>(workspace);
  float* w27 = x27 + (size_t)P * 32;
  const int round = precise() ? 0 : 1;
  im2col_first_kernel<<<grid_1d((size_t)P, 128), 128, 0, stream>>>(x_nchw, x27, N, H, W, round);
  HK_LAUNCH_CHECK("im2col_first_kernel");
  pack_first_weights_kernel<<<(Cout * 32 + 127) / 128, 128, 0, stream>>>(w, bias, w27, Cout, round);
  HK_LAUNCH_CHECK("pack_first_weights_kernel");
  GemmEpi e = {};
  e.C = y_nhwc; e.ldc = Cout; e.alpha = 1.f;
  e.relu = 3;                                        // ReLU + tf32 rounding
  return gemm_tf32(x27, 0, 32, 0, w27, 0, 32, 0, e, (int)P, Cout, 32, 1, stream);
}

static int first_wgrad_splits(long long P) {
  for (int S = 592; S > 1; --S)
    if (P % S == 0) return S;
  return 1;
}

size_t hk_conv3x3_first_wgrad_workspace_bytes(int N, int H, int W, int Cout) {
  return (size_t)first_wgrad_splits((long long)N * H * W) * Cout * 32 * sizeof(float);
}

/* dw [Cout,3,3,3], db [Cout] of the input layer from X27 (written by hk_conv3x3_first_fwd) and dy (ReLU-masked):
 * split-K batched MN-major wgmma GEMM  partial[s] = dY_s^T . X27_s ; column 27 of the result is the bias grad. */
int hk_conv3x3_first_wgrad_acc(const float* x27, const float* dy_nhwc, float* dw, float* db, int N, int H, int W, int Cout,
                               void* workspace, size_t workspace_bytes, int accumulate, void* stream_);
int hk_conv3x3_first_wgrad(const float* x27, const float* dy_nhwc, float* dw, float* db, int N, int H, int W,
                           int Cout, void* workspace, size_t workspace_bytes, void* stream_) {
  return hk_conv3x3_first_wgrad_acc(x27, dy_nhwc, dw, db, N, H, W, Cout, workspace, workspace_bytes, 0, stream_);
}
int hk_conv3x3_first_wgrad_acc(const float* x27, const float* dy_nhwc, float* dw, float* db, int N, int H, int W, int Cout,
                               void* workspace, size_t workspace_bytes, int accumulate, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  HK_REQUIRE(x27 && dy_nhwc && dw, HK_ERR_ARG, "hk_conv3x3_first_wgrad: null pointer");
  HK_REQUIRE(Cout % 4 == 0 && Cout <= 128, HK_ERR_UNSUPPORTED, "hk_conv3x3_first_wgrad: Cout=%d unsupported", Cout);
  HK_REQUIRE(workspace && workspace_bytes >= hk_conv3x3_first_wgrad_workspace_bytes(N, H, W, Cout), HK_ERR_WORKSPACE,
             "hk_conv3x3_first_wgrad: workspace too small");
  const long long P = (long long)N * H * W;
  const int S = first_wgrad_splits(P);
  float* part = static_cast<float*>(workspace);
  // partial columns 0..26 are dw[co][27]; column 27 (the ones column of X27) is db
  int r = gemm_splitk(dy_nhwc, 1, Cout, x27, 1, 32, Cout, 32, P, S, part, dw, 27, 27, nullptr, accumulate, stream);
  if (r || !db) return r;
  return sum_splits(part + 27, S, (long long)Cout * 32, Cout, 1, 32, db, 1, nullptr, accumulate, stream);
}

int hk_conv3x3_first_fwd_direct(const float* x_nchw, const float* w, const float* bias, float* y_nhwc, int N, int H, int W,
                                int Cout, void* stream) {
  HK_REQUIRE(!precise(), HK_ERR_UNSUPPORTED, "hk_conv3x3_first_fwd_direct: not available in 3xTF32 mode");
  HK_REQUIRE(x_nchw && w && y_nhwc, HK_ERR_ARG, "hk_conv3x3_first_fwd_direct: null pointer");
  HK_REQUIRE(Cout == 64, HK_ERR_UNSUPPORTED, "hk_conv3x3_first_fwd_direct: Cout=%d unsupported (64 only)", Cout);
  HK_REQUIRE(N > 0 && H > 0 && W > 0, HK_ERR_ARG, "hk_conv3x3_first_fwd_direct: empty map");
  HK_REQUIRE((reinterpret_cast<uintptr_t>(y_nhwc) & 7) == 0, HK_ERR_ALIGN, "hk_conv3x3_first_fwd_direct: y not 8-byte aligned");
  const long long P = (long long)N * H * W;
  HK_REQUIRE(P < (1ll << 31), HK_ERR_UNSUPPORTED, "hk_conv3x3_first_fwd_direct: too many pixels");
  first_fwd_direct_kernel<<<(int)((P + FIRST_FWD_PIX - 1) / FIRST_FWD_PIX), 128, FIRST_FWD_SMEM, (cudaStream_t)stream>>>(
      x_nchw, w, bias, y_nhwc, N, H, W);
  HK_LAUNCH_CHECK("first_fwd_direct_kernel");
  return 0;
}

static int first_wgrad_direct_ctas() { return 2 * num_sms(); }   // two CTAs per SM (launch bounds)

size_t hk_conv3x3_first_wgrad_direct_workspace_bytes(void) {
  return (size_t)first_wgrad_direct_ctas() * 64 * 32 * sizeof(float);
}

int hk_conv3x3_first_wgrad_direct_acc(const float* x_nchw, const float* dy_nhwc, float* dw, float* db, int N, int H, int W,
                                      int Cout, void* workspace, size_t workspace_bytes, int accumulate, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  HK_REQUIRE(!precise(), HK_ERR_UNSUPPORTED, "hk_conv3x3_first_wgrad_direct: not available in 3xTF32 mode");
  HK_REQUIRE(x_nchw && dy_nhwc && dw, HK_ERR_ARG, "hk_conv3x3_first_wgrad_direct: null pointer");
  HK_REQUIRE(Cout == 64, HK_ERR_UNSUPPORTED, "hk_conv3x3_first_wgrad_direct: Cout=%d unsupported (64 only)", Cout);
  HK_REQUIRE(N > 0 && H > 0 && W > 0, HK_ERR_ARG, "hk_conv3x3_first_wgrad_direct: empty map");
  HK_REQUIRE(workspace && workspace_bytes >= hk_conv3x3_first_wgrad_direct_workspace_bytes(), HK_ERR_WORKSPACE,
             "hk_conv3x3_first_wgrad_direct: workspace too small");
  HK_REQUIRE((long long)N * H * W < (1ll << 31), HK_ERR_UNSUPPORTED, "hk_conv3x3_first_wgrad_direct: too many pixels");
  const int G = first_wgrad_direct_ctas();
  float* part = static_cast<float*>(workspace);
  first_wgrad_direct_kernel<<<G, FIRST_WG_THREADS, FIRST_WG_SMEM, stream>>>(x_nchw, dy_nhwc, part, N, H, W);
  HK_LAUNCH_CHECK("first_wgrad_direct_kernel");
  // partial columns 0..26 are dw[co][27]; column 27 (the ones column of X27) is db
  int r = sum_splits(part, G, 64 * 32, 64, 27, 32, dw, 27, nullptr, accumulate, stream);
  if (r || !db) return r;
  return sum_splits(part + 27, G, 64 * 32, 64, 1, 32, db, 1, nullptr, accumulate, stream);
}

int hk_maxpool2x2_fwd(const float* x_nhwc, float* y, int N, int H, int W, int C, int out_nchw, void* stream) {
  HK_REQUIRE(x_nhwc && y, HK_ERR_ARG, "hk_maxpool2x2_fwd: null pointer");
  HK_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, HK_ERR_UNSUPPORTED, "hk_maxpool2x2_fwd: C%%4, even H/W required");
  const size_t total = (size_t)N * (H / 2) * (W / 2) * (C / 4);
  maxpool2x2_fwd_kernel<<<grid_1d(total, 256), 256, 0, (cudaStream_t)stream>>>(x_nhwc, y, N, H, W, C, out_nchw);
  HK_LAUNCH_CHECK("maxpool2x2_fwd_kernel");
  return 0;
}

int hk_maxpool2x2_bwd(const float* x_nhwc, const float* dy, float* dx_nhwc, int N, int H, int W, int C, int dy_nchw,
                      void* stream) {
  HK_REQUIRE(x_nhwc && dy && dx_nhwc, HK_ERR_ARG, "hk_maxpool2x2_bwd: null pointer");
  HK_REQUIRE(H % 2 == 0 && W % 2 == 0, HK_ERR_UNSUPPORTED, "hk_maxpool2x2_bwd: even H/W required");
  const size_t total = (size_t)N * (H / 2) * (W / 2) * C;
  maxpool2x2_bwd_kernel<<<grid_1d(total, 256), 256, 0, (cudaStream_t)stream>>>(x_nhwc, dy, dx_nhwc, N, H, W, C, dy_nchw);
  HK_LAUNCH_CHECK("maxpool2x2_bwd_kernel");
  return 0;
}

int hk_maxpool2x2_fwd_idx(const float* x_nhwc, float* y, unsigned char* code, int N, int H, int W, int C, int out_nchw,
                          void* stream) {
  HK_REQUIRE(x_nhwc && y && code, HK_ERR_ARG, "hk_maxpool2x2_fwd_idx: null pointer");
  HK_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, HK_ERR_UNSUPPORTED, "hk_maxpool2x2_fwd_idx: C%%4, even H/W required");
  const size_t total = (size_t)N * (H / 2) * (W / 2) * (C / 4);
  maxpool2x2_fwd_idx_kernel<<<grid_1d(total, 256), 256, 0, (cudaStream_t)stream>>>(x_nhwc, y, code, N, H, W, C, out_nchw);
  HK_LAUNCH_CHECK("maxpool2x2_fwd_idx_kernel");
  return 0;
}

int hk_maxpool2x2_bwd_idx(const unsigned char* code, const float* dy, float* dx_nhwc, int N, int H, int W, int C,
                          int dy_nchw, void* stream) {
  HK_REQUIRE(code && dy && dx_nhwc, HK_ERR_ARG, "hk_maxpool2x2_bwd_idx: null pointer");
  HK_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, HK_ERR_UNSUPPORTED, "hk_maxpool2x2_bwd_idx: C%%4, even H/W required");
  const size_t total = (size_t)N * (H / 2) * (W / 2) * (C / 4);
  maxpool2x2_bwd_idx_kernel<<<grid_1d(total, 256), 256, 0, (cudaStream_t)stream>>>(code, dy, dx_nhwc, N, H, W, C, dy_nchw);
  HK_LAUNCH_CHECK("maxpool2x2_bwd_idx_kernel");
  return 0;
}

}  // extern "C"
