// Generic batched TF32 GEMM on wgmma (sm_90a) with TMA-fed, 128B-swizzled shared-memory operands and the fp32
// accumulator in registers.  One 128 x BN output tile per CTA iteration.
//
//   C[b] = alpha_b * (A[b] . B[b]) + diag * I + beta_b * D[b]           (optionally stored transposed)
//
// Both operands may be K-major or MN-major in global memory, so the same kernel serves
//   * Newton-Schulz chains and covariance of Fast MPN-COV (reference model/methods/MPNCOV.py:105-202),
//   * the Gram and (S . X) contractions of the bilinear / compact-bilinear pooling (BCNN.py:13-27, CBCNN.py:96-135),
//   * 1x1 convolutions in NHWC (model/backbone/resnet.py:29-37).
// tf32 wgmma reads K-major operands only: an MN-major operand is TMA-loaded into a staging buffer and transposed into
// the K-major stage by the producer warpgroup.
// Warp roles: warpgroup 0 = producer (warp 0 lane 0 issues TMA; all four warps transpose MN-major tiles),
// warpgroups 1-2 = MMA + epilogue, rows 0-63 and 64-127 of the tile.
#include <stdlib.h>

#include "common.cuh"
#include "host.h"
#include "gemm.h"
#include "../../include/hawkeye_b200.h"

namespace hk {

constexpr int GEMM_THREADS = 384;
constexpr int GEMM_SMEM_MAX = 227 * 1024;   // largest dynamic shared memory a block may opt in to on sm_90

template <int BN>
struct GemmCfg {
  static constexpr int STAGES = 4;
  static constexpr int A_BYTES = 128 * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RAW_BYTES = A_BYTES + B_BYTES;    // staging of MN-major operands (one k-block, hi or lo)
  static constexpr int ACC_TILE = 2 * 128 * 33 * 4;      // two 32-column accumulator chunks, row-major, padded rows
  static constexpr int EPI_TILE = 4 * 32 * 36 * 4;       // four epilogue warps x a 32 x 36-float transpose tile
  static constexpr int SMEM_FIXED = 1024 /*align slack*/ + 256 /*barriers*/ + ACC_TILE + 2 * EPI_TILE;
};

// Persistent: one CTA per SM walks output tiles t, t+grid, ... (n-tile fastest, so CTAs running at the same time share
// the A rows through L2).  The smem ring runs across tile boundaries, so the producer loads tile i+1 while the consumers
// finish tile i.  The epilogue stages each pair of 32-column accumulator chunks through shared memory, after which
// consumer thread (half, q, lane) owns row 32 q + lane of chunk 2 c + half.
template <int BN, bool TRIPLE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
wgmma_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmAl, const __grid_constant__ CUtensorMap tmBl, GemmEpi epi,
                  int M, int N, int K, int a_mn, int b_mn, int shareA, int shareB, int nstages,
                  int tiles_m, int tiles_n, int total_tiles) {
  // triple: operands are (hi, lo) tf32 pairs (tmA/tmB = hi, tmAl/tmBl = lo) and every k-step issues Ah.Bl, Al.Bh, Ah.Bh
  // — the 3xTF32 product of the Newton-Schulz chain in ONE launch, no partial sums through memory
  using Cfg = GemmCfg<BN>;
  constexpr int NACC = BN / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int nops = TRIPLE ? 2 : 1;
  uint8_t* sA = smem;
  uint8_t* sB = smem + nstages * Cfg::A_BYTES;
  uint8_t* sAl = smem + nstages * Cfg::STAGE_BYTES;
  uint8_t* sBl = sAl + nstages * Cfg::A_BYTES;
  const bool any_mn = a_mn || b_mn;
  uint8_t* raw = smem + nstages * Cfg::STAGE_BYTES * nops;                  // [nops][A_BYTES + B_BYTES] when any_mn
  uint8_t* after = raw + (any_mn ? nops * Cfg::RAW_BYTES : 0);
  uint64_t* full = reinterpret_cast<uint64_t*>(after);
  uint64_t* empty = full + nstages;
  uint64_t* raw_bar = empty + nstages;
  float* acc_tile = reinterpret_cast<float*>(after + 256);
  float* epi_tiles = acc_tile + Cfg::ACC_TILE / 4;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nk = (K + 31) / 32;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < nstages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);
    }
    mbar_init(raw_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ---------------------------------------------------------------- producer warpgroup
    regs_dealloc<56>();
    const int t = threadIdx.x;
    int kbg = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int nt = tile % tiles_n;
      const int mt = (tile / tiles_n) % tiles_m;
      const int bz = tile / (tiles_n * tiles_m);
      const int m0 = mt * 128, n0 = nt * BN;
      const int bza = shareA ? 0 : bz, bzb = shareB ? 0 : bz;
      for (int kb = 0; kb < nk; ++kb, ++kbg) {
        const int s = kbg % nstages;
        const uint32_t ph = (kbg / nstages) & 1;
        if (t == 0) {
          mbar_wait(&empty[s], ph ^ 1);
          // K-major operands go straight into the stage; MN-major ones into the staging buffer
          uint32_t direct = 0, staged = 0;
          for (int o = 0; o < nops; ++o) {
            (a_mn ? staged : direct) += Cfg::A_BYTES;
            (b_mn ? staged : direct) += Cfg::B_BYTES;
          }
          if (!any_mn) mbar_expect_tx(&full[s], direct);
          else mbar_expect_tx(raw_bar, direct + staged);
          uint64_t* bar = any_mn ? raw_bar : &full[s];
          for (int o = 0; o < nops; ++o) {
            const CUtensorMap* ma = o ? &tmAl : &tmA;
            const CUtensorMap* mb = o ? &tmBl : &tmB;
            uint8_t* a = (o ? sAl : sA) + s * Cfg::A_BYTES;
            uint8_t* b = (o ? sBl : sB) + s * Cfg::B_BYTES;
            uint8_t* ra = raw + o * Cfg::RAW_BYTES;
            uint8_t* rb = ra + Cfg::A_BYTES;
            if (!a_mn) {
              tma_load_3d(a, ma, bar, kb * 32, m0, bza);
            } else {
#pragma unroll
              for (int j = 0; j < 4; ++j) tma_load_3d(ra + j * 4096, ma, bar, m0 + j * 32, kb * 32, bza);
            }
            if (!b_mn) {
              tma_load_3d(b, mb, bar, kb * 32, n0, bzb);
            } else {
#pragma unroll
              for (int j = 0; j < BN / 32; ++j) tma_load_3d(rb + j * 4096, mb, bar, n0 + j * 32, kb * 32, bzb);
            }
          }
        }
        if (any_mn) {
          mbar_wait(raw_bar, kbg & 1);
          for (int o = 0; o < nops; ++o) {
            const uint8_t* ra = raw + o * Cfg::RAW_BYTES;
            if (a_mn) transpose_mn_tile(ra, (o ? sAl : sA) + s * Cfg::A_BYTES, 128, t, 128);
            if (b_mn) transpose_mn_tile(ra + Cfg::A_BYTES, (o ? sBl : sB) + s * Cfg::B_BYTES, BN, t, 128);
          }
          fence_proxy_async();       // generic-proxy stores -> visible to wgmma (async proxy)
          named_bar(1, 128);         // whole staging buffer consumed before the next TMA overwrites it
          if (t == 0) mbar_arrive(&full[s]);
        }
      }
    }
  } else {
    // ---------------------------------------------------------------- consumers: MMA, then epilogue
    regs_alloc<224>();
    const int ct = threadIdx.x - 128;          // 0..255
    const int wg = ct >> 7;                    // row half of the tile this warpgroup multiplies
    const int half = ct >> 7;                  // accumulator chunk parity this thread stores in the epilogue
    const int q = (ct >> 5) & 3;
    const int wl = (ct & 127) >> 5;            // warp within the warpgroup (fragment rows 16 wl ..)
    int kbg = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int nt = tile % tiles_n;
      const int mt = (tile / tiles_n) % tiles_m;
      const int bz = tile / (tiles_n * tiles_m);
      const int m0 = mt * 128, n0 = nt * BN;
      float acc[NACC], acc2[TRIPLE ? NACC : 1];
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
      if constexpr (TRIPLE) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc2[i] = 0.f;
      }
      // triple mode keeps TWO accumulators — the leading product Ah.Bh and the sum of the two correction products — added
      // in the epilogue, so the small correction terms are not lost against the running sum
      for (int kb = 0; kb < nk; ++kb, ++kbg) {
        const int s = kbg % nstages;
        const uint32_t ph = (kbg / nstages) & 1;
        mbar_wait(&full[s], ph);
        const uint64_t a_base = make_sdesc(smem_u32(sA + s * Cfg::A_BYTES + wg * 64 * 128));
        const uint64_t b_base = make_sdesc(smem_u32(sB + s * Cfg::B_BYTES));
        wgmma_fence();
        if constexpr (TRIPLE) {
          const uint64_t al_base = make_sdesc(smem_u32(sAl + s * Cfg::A_BYTES + wg * 64 * 128));
          const uint64_t bl_base = make_sdesc(smem_u32(sBl + s * Cfg::B_BYTES));
          // a partial last k-block is zero-filled by TMA past K: all four k-steps run, keeping the wgmma stream uniform
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            wgmma_tf32(acc2, a_base + ks * 2, bl_base + ks * 2, 1);
            wgmma_tf32(acc2, al_base + ks * 2, b_base + ks * 2, 1);
            wgmma_tf32(acc, a_base + ks * 2, b_base + ks * 2, 1);
          }
        } else {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) wgmma_tf32(acc, a_base + ks * 2, b_base + ks * 2, 1);
        }
        wgmma_commit();
        // one group stays in flight: the MMAs of k-block kb overlap the wait for kb + 1; the stage of kb - 1 is released
        wgmma_wait<1>();
        wgmma_keep(acc);
        if constexpr (TRIPLE) wgmma_keep(acc2);
        if (kb > 0 && (ct & 127) == 0) mbar_arrive(&empty[(kbg - 1) % nstages]);
      }
      wgmma_wait<0>();
      wgmma_keep(acc);
      if constexpr (TRIPLE) wgmma_keep(acc2);
      if ((ct & 127) == 0) mbar_arrive(&empty[(kbg - 1) % nstages]);
      if constexpr (TRIPLE) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] += acc2[i];
      }
      const int row = m0 + q * 32 + lane;
      // post_scale: the value becomes sqrt(alpha_b * acc + post_eps) * post_scale[b] before the rest of the epilogue
      const float alpha_b = epi.alpha * (epi.alpha_vec ? epi.alpha_vec[bz] : 1.f);
      const float pscale = epi.post_scale ? epi.post_scale[bz] : 0.f;
      const float alpha = epi.post_scale ? 1.f : alpha_b;
      const float beta = epi.beta * (epi.beta_vec ? epi.beta_vec[bz] : 1.f);
      float* Cb = epi.C + (long long)bz * epi.strideC;
      const float* Db = epi.D ? epi.D + (long long)bz * epi.strideD : nullptr;
      const float* Dlb = (epi.D && epi.D_lo) ? epi.D_lo + (long long)bz * epi.strideD : nullptr;
      const long long ldE = epi.ldE ? epi.ldE : epi.ldc;
      const float* Eb = epi.E ? epi.E + (long long)bz * (epi.ldE ? epi.strideE : epi.strideC) : nullptr;
      float* Clb = epi.C_lo ? epi.C_lo + (long long)bz * epi.strideC : nullptr;
      const bool simple = !Eb && !Clb && !Dlb && epi.diag == 0.f && !epi.trans_c && (!Db || epi.ldd != 0) && !epi.mode;
      float cr = 0.f;                          // EPI_BILINEAR_S: this thread's share of <dY, z>
#pragma unroll
      for (int cp = 0; cp < BN / 64; ++cp) {
        // fragments of chunks 2 cp, 2 cp + 1 -> acc_tile[chunk parity][row][33]
        named_bar(2, 256);
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
        named_bar(2, 256);
        const int c = 2 * cp + half;
        float v[32];
        {
          const float* src = acc_tile + half * (128 * 33) + (q * 32 + lane) * 33;
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = src[j];
        }
        if (epi.post_scale) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = sqrtf(fmaf(v[j], alpha_b, epi.post_eps)) * pscale;
        }
        if (epi.mode == EPI_BILINEAR_S) {
          const int col0 = n0 + c * 32;
          if (row < M && col0 < N) {
            const float* dyb = epi.dY + (long long)bz * M * N;
            const float* drow = dyb + (long long)row * N + col0;
            float* dst = Cb + (long long)row * epi.ldc + col0;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              if (col0 + j < N) {
                const float z = sqrtf(fmaf(v[j], alpha_b, epi.post_eps));
                const float dv = drow[j];
                cr = fmaf(dv, z, cr);
                // dY[j][i]: for a fixed j the lanes of the warp hold consecutive rows i — one coalesced 128 B read
                dst[j] = (dv + dyb[(long long)(col0 + j) * N + row]) / (2.f * z);
              }
            }
          }
          continue;
        }
        if (epi.mode == EPI_SKETCH) {
          const int col0 = n0 + c * 32;
          if (row < M && col0 < N) {
            float* bins = epi.bins + (long long)bz * epi.d;
            const int hi = epi.h1[row];
            const float si = epi.s1[row] * alpha_b;
#pragma unroll 4
            for (int j = 0; j < 32; ++j) {
              if (col0 + j < N) {
                int k = hi + __ldg(epi.h2 + col0 + j);
                if (k >= epi.d) k -= epi.d;
                atomicAdd(bins + k, si * __ldg(epi.s2 + col0 + j) * v[j]);
              }
            }
          }
          continue;
        }
        const int col0 = n0 + c * 32;
        // fast path (plain scaled store of a full, aligned 32-column chunk): a handful of instructions per element — the
        // general path below costs ~60 and dominates short-K GEMMs such as the first VGG layer (K = 32)
        if (simple && col0 + 32 <= N && (epi.ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(Cb) & 15) == 0 &&
            (!Db || ((epi.ldd & 3) == 0 && (reinterpret_cast<uintptr_t>(Db) & 15) == 0))) {
          // A thread owns 32 consecutive columns of ONE row, so a direct float4 store instruction would touch 32 rows x 16 B —
          // half-written 32 B sectors, twice the L2 write transactions (the 1x1-conv GEMMs of the ResNet trunk are
          // output-write-bound).  Transpose the 32 x 32 chunk through a warp-private shared-memory tile instead: every store
          // instruction then writes four full 128 B rows; the optional addend D (residual gradient) is read the same way.
          float* tile = epi_tiles + (ct >> 5) * (32 * 36);
#pragma unroll
          for (int j = 0; j < 32; j += 4)
            *reinterpret_cast<float4*>(tile + lane * 36 + j) =
                make_float4(alpha * v[j], alpha * v[j + 1], alpha * v[j + 2], alpha * v[j + 3]);
          __syncwarp();
          const int row0 = m0 + q * 32;
          float4 dadd[8];
          if (Db) {      // all eight addend loads in flight before the first store (C and D may alias as far as the compiler knows)
#pragma unroll
            for (int it = 0; it < 8; ++it) {
              const int r = it * 4 + (lane >> 3);
              dadd[it] = (row0 + r < M) ? __ldg(reinterpret_cast<const float4*>(Db + (long long)(row0 + r) * epi.ldd + col0 + (lane & 7) * 4))
                                        : make_float4(0.f, 0.f, 0.f, 0.f);
            }
          }
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            const int r = it * 4 + (lane >> 3);
            float4 t = *reinterpret_cast<const float4*>(tile + r * 36 + (lane & 7) * 4);
            if (row0 + r < M) {
              if (Db) {
                const float4 d = dadd[it];
                t.x = fmaf(beta, d.x, t.x); t.y = fmaf(beta, d.y, t.y); t.z = fmaf(beta, d.z, t.z); t.w = fmaf(beta, d.w, t.w);
              }
              if (epi.relu & 1) { t.x = fmaxf(t.x, 0.f); t.y = fmaxf(t.y, 0.f); t.z = fmaxf(t.z, 0.f); t.w = fmaxf(t.w, 0.f); }
              if (epi.relu & 2) { t.x = tf32_round(t.x); t.y = tf32_round(t.y); t.z = tf32_round(t.z); t.w = tf32_round(t.w); }
              *reinterpret_cast<float4*>(Cb + (long long)(row0 + r) * epi.ldc + col0 + (lane & 7) * 4) = t;
            }
          }
          __syncwarp();
          continue;
        }
        if (row < M && col0 < N) {
          // general epilogue: raw addend E, alpha, diagonal, beta*(D [+ D_lo]), ReLU / rounding, plain / (hi, lo) / transposed
          // store.  A thread owns 32 consecutive columns of one row: whole aligned chunks move as float4 (the Newton-Schulz
          // chain lives on this path; scalar accesses made its epilogues 3-8x longer than the MMAs)
          const bool full = col0 + 32 <= N;
          const float* ep = Eb ? Eb + (long long)row * ldE + col0 : nullptr;
          const float* dp = Db ? Db + (long long)row * epi.ldd + col0 : nullptr;
          const float* dlp = Dlb ? Dlb + (long long)row * epi.ldd + col0 : nullptr;
          auto vec_ok = [&](const void* q) { return full && (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
          if (ep) {
            if (vec_ok(ep)) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                const float4 t = *reinterpret_cast<const float4*>(ep + j);
                v[j] += t.x; v[j + 1] += t.y; v[j + 2] += t.z; v[j + 3] += t.w;
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (col0 + j < N) v[j] += ep[j];
            }
          }
          float dv[32];
          if (dp) {
            if (vec_ok(dp) && (!dlp || vec_ok(dlp))) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                float4 t = *reinterpret_cast<const float4*>(dp + j);
                if (dlp) {
                  const float4 u = *reinterpret_cast<const float4*>(dlp + j);
                  t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
                }
                dv[j] = t.x; dv[j + 1] = t.y; dv[j + 2] = t.z; dv[j + 3] = t.w;
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                dv[j] = 0.f;
                if (col0 + j < N) dv[j] = dp[j] + (dlp ? dlp[j] : 0.f);
              }
            }
          }
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            float o = alpha * v[j];
            if (col0 + j == row) o += epi.diag;
            if (dp) o += beta * dv[j];
            if (epi.relu & 1) o = fmaxf(o, 0.f);
            if (epi.relu & 2) o = tf32_round(o);   // output feeds another tf32 MMA: keep its error unbiased
            v[j] = o;
          }
          if (Clb) {   // (hi, lo) split store; not combined with trans_c
            float* hp = Cb + (long long)row * epi.ldc + col0;
            float* lp = Clb + (long long)row * epi.ldc + col0;
            if (vec_ok(hp) && vec_ok(lp)) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                const float h0 = tf32_round(v[j]), h1 = tf32_round(v[j + 1]), h2 = tf32_round(v[j + 2]), h3 = tf32_round(v[j + 3]);
                *reinterpret_cast<float4*>(hp + j) = make_float4(h0, h1, h2, h3);
                *reinterpret_cast<float4*>(lp + j) = make_float4(tf32_round(v[j] - h0), tf32_round(v[j + 1] - h1),
                                                                 tf32_round(v[j + 2] - h2), tf32_round(v[j + 3] - h3));
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j) {
                const float hi = tf32_round(v[j]);
                if (col0 + j < N) { hp[j] = hi; lp[j] = tf32_round(v[j] - hi); }
              }
            }
          } else if (!epi.trans_c) {
            float* dst = Cb + (long long)row * epi.ldc + col0;
            if (vec_ok(dst)) {
#pragma unroll
              for (int j = 0; j < 32; j += 4)
                *reinterpret_cast<float4*>(dst + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (col0 + j < N) dst[j] = v[j];
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (col0 + j < N) Cb[(long long)(col0 + j) * epi.ldc + row] = v[j];
          }
        }
      }
      if (epi.mode == EPI_BILINEAR_S) {        // fp64 atomics: the image's sum does not depend on their order at fp32 level
        cr = warp_sum(cr);
        if (lane == 0) atomicAdd(epi.c_raw + bz, (double)cr);
      }
    }
  }
}

static int make_operand_map(CUtensorMap* tm, const float* P, int mn_major, long long ld, long long stride, int rows,
                            int K, int batch, int tile_rows, int* share) {
  *share = (stride == 0 || batch == 1);
  uint64_t dims[3], strides[2];
  uint32_t box[3];
  const uint64_t nb = *share ? 1 : (uint64_t)batch;
  const uint64_t bs = *share ? (uint64_t)(mn_major ? K : rows) * ld * 4 : (uint64_t)stride * 4;
  if (!mn_major) {  // [rows][K], K contiguous
    dims[0] = K; dims[1] = rows; dims[2] = nb;
    box[0] = 32; box[1] = tile_rows; box[2] = 1;
  } else {          // [K][rows], rows contiguous
    dims[0] = rows; dims[1] = K; dims[2] = nb;
    box[0] = 32; box[1] = 32; box[2] = 1;
  }
  strides[0] = (uint64_t)ld * 4;
  strides[1] = bs;
  return make_tmap(tm, P, 3, dims, strides, box);
}

template <int BN>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmEpi& epi, int M, int N, int K,
                       int batch, int a_mn, int b_mn, int shareA, int shareB, cudaStream_t stream,
                       const CUtensorMap* tmAl = nullptr, const CUtensorMap* tmBl = nullptr) {
  using Cfg = GemmCfg<BN>;
  if (int r = allow_dynamic_smem<wgmma_gemm_kernel<BN, false>>(GEMM_SMEM_MAX, BN == 64 ? "gemm<64>" : "gemm<128>")) return r;
  if constexpr (BN == 64)
    if (int r = allow_dynamic_smem<wgmma_gemm_kernel<64, true>>(GEMM_SMEM_MAX, "gemm<64>")) return r;
  const int tiles_m = (M + 127) / 128, tiles_n = (N + BN - 1) / BN;
  const long long total = (long long)tiles_m * tiles_n * batch;
  if (total >= (1ll << 31)) return set_error(HK_ERR_UNSUPPORTED, "gemm: too many tiles");
  const int sms = num_sms();
  const int nk = (K + 31) / 32;
  const long long kblocks_per_cta = (long long)nk * ((total + sms - 1) / sms);
  const int triple = tmAl ? 1 : 0;
  const int nops = triple ? 2 : 1;
  const int raw = (a_mn || b_mn) ? nops * Cfg::RAW_BYTES : 0;
  int max_stages = (GEMM_SMEM_MAX - Cfg::SMEM_FIXED - raw) / (Cfg::STAGE_BYTES * nops);   // what fits in 227 KB
  if (max_stages > Cfg::STAGES) max_stages = Cfg::STAGES;
  const int nstages = kblocks_per_cta < max_stages ? (int)kblocks_per_cta : max_stages;
  const int smem = nstages * Cfg::STAGE_BYTES * nops + raw + Cfg::SMEM_FIXED;
  const int grid = total < sms ? (int)total : sms;
  bool launched = false;
  if constexpr (BN == 64) {   // the 3xTF32 pair kernel runs 64-wide tiles only (two accumulators per thread)
    if (triple) {
      wgmma_gemm_kernel<64, true><<<grid, GEMM_THREADS, smem, stream>>>(tmA, tmB, *tmAl, *tmBl, epi, M, N, K, a_mn, b_mn, shareA,
                                                                        shareB, nstages, tiles_m, tiles_n, (int)total);
      launched = true;
    }
  }
  if (!launched)
    wgmma_gemm_kernel<BN, false><<<grid, GEMM_THREADS, smem, stream>>>(tmA, tmB, tmA, tmB, epi, M, N, K, a_mn, b_mn, shareA,
                                                                       shareB, nstages, tiles_m, tiles_n, (int)total);
  HK_LAUNCH_CHECK("wgmma_gemm_kernel");
  return 0;
}

__global__ void tf32_split_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    const float h = tf32_round(v);
    if (hi) hi[i] = h;
    if (lo) lo[i] = tf32_round(v - h);
  }
}

int tf32_split(const float* x, float* hi, float* lo, size_t n, cudaStream_t stream) {
  if (!n) return 0;
  tf32_split_kernel<<<grid_1d(n, 256), 256, 0, stream>>>(x, hi, lo, n);
  HK_LAUNCH_CHECK("tf32_split_kernel");
  return 0;
}

// floats spanned by a strided operand: `batch` matrices of `rows` x `cols` (cols contiguous), leading dimension ld
static size_t operand_extent(long long rows, long long cols, long long ld, long long stride, int batch) {
  return (size_t)((long long)(batch - 1) * (stride > 0 ? stride : 0) + (rows - 1) * ld + cols);
}

// What the TMA-fed kernel needs of an operand, checked before any scratch allocation, driver call or launch so that a
// rejected call launches nothing in either precision mode: a 16-byte aligned base, and a row pitch and (used) batch
// stride that are whole 16-byte units.
static int check_operand(const char* what, char name, const float* P, long long ld, long long stride, int batch) {
  HK_REQUIRE(P, HK_ERR_ARG, "%s: null operand %c", what, name);
  HK_REQUIRE(aligned16(P), HK_ERR_ALIGN, "%s: operand %c is not 16-byte aligned", what, name);
  HK_REQUIRE(ld > 0 && ld % 4 == 0, HK_ERR_ALIGN, "%s: ld%c=%lld is not a positive multiple of 4 floats (16-byte stride)",
             what, name, ld);
  HK_REQUIRE(batch == 1 || stride % 4 == 0, HK_ERR_ALIGN,
             "%s: batch stride of %c (%lld) is not a multiple of 4 floats (16-byte stride)", what, name, stride);
  return 0;
}

static int check_gemm_args(const char* what, const float* A, long long lda, long long strideA, const float* B,
                           long long ldb, long long strideB, const GemmEpi& epi, int M, int N, int K, int batch) {
  HK_REQUIRE(epi.C, HK_ERR_ARG, "%s: null output", what);
  HK_REQUIRE(M > 0 && N > 0 && K > 0 && batch > 0, HK_ERR_ARG, "%s: bad shape M=%d N=%d K=%d batch=%d", what, M, N, K,
             batch);
  HK_REQUIRE(batch <= 65535, HK_ERR_UNSUPPORTED, "%s: batch %d > 65535", what, batch);
  if (int r = check_operand(what, 'a', A, lda, strideA, batch)) return r;
  return check_operand(what, 'b', B, ldb, strideB, batch);
}

// 3xTF32: A.B ~= Ah.Bh + Al.Bh + Ah.Bl with (hi, lo) = tf32 halves of the operands, split into scratch and multiplied
// by ONE launch of the pair kernel, so the caller's epilogue (alpha, diag, D, ReLU, transposed store ...) is applied
// once, to the full sum.
int gemm_tf32_3x(const float* A, int a_mn, long long lda, long long strideA, const float* B, int b_mn, long long ldb,
                        long long strideB, const GemmEpi& epi, int M, int N, int K, int batch, cudaStream_t st) {
  if (int r = check_gemm_args("gemm (3xTF32)", A, lda, strideA, B, ldb, strideB, epi, M, N, K, batch)) return r;
  const size_t nA = operand_extent(a_mn ? K : M, a_mn ? M : K, lda, strideA, batch);
  const bool same = (A == B && a_mn == b_mn && lda == ldb && strideA == strideB && M == N);
  const size_t nB = same ? 0 : operand_extent(b_mn ? K : N, b_mn ? N : K, ldb, strideB, batch);
  const size_t nA4 = (nA + 3) & ~size_t(3), nB4 = (nB + 3) & ~size_t(3);     // the lo halves start 16-byte aligned (TMA)
  Scratch sa(2 * nA4 * sizeof(float), st), sb(2 * (nB4 ? nB4 : 4) * sizeof(float), st);
  HK_REQUIRE(sa.p && sb.p, HK_ERR_DRIVER, "gemm (precise): cudaMallocAsync of the operand halves failed");
  float *Ah = sa.f(), *Al = Ah + nA4;
  float *Bh = same ? Ah : sb.f(), *Bl = same ? Al : Bh + nB4;
  int r;
  if ((r = tf32_split(A, Ah, Al, nA, st))) return r;
  if (!same && (r = tf32_split(B, Bh, Bl, nB, st))) return r;
  GemmEpi f = epi;
  f.relu &= ~2;                                                                                             // no rounding
  return gemm_tf32_pair(Ah, Al, a_mn, lda, strideA, Bh, Bl, b_mn, ldb, strideB, f, M, N, K, batch, st);     // one launch
}

int gemm_tf32(const float* A, int a_mn, long long lda, long long strideA, const float* B, int b_mn, long long ldb,
              long long strideB, const GemmEpi& epi, int M, int N, int K, int batch, cudaStream_t stream) {
  if (precise()) return gemm_tf32_3x(A, a_mn, lda, strideA, B, b_mn, ldb, strideB, epi, M, N, K, batch, stream);
  return gemm_tf32_1x(A, a_mn, lda, strideA, B, b_mn, ldb, strideB, epi, M, N, K, batch, stream);
}

int gemm_tf32_1x(const float* A, int a_mn, long long lda, long long strideA, const float* B, int b_mn, long long ldb,
                 long long strideB, const GemmEpi& epi, int M, int N, int K, int batch, cudaStream_t stream) {
  if (int r = check_gemm_args("gemm", A, lda, strideA, B, ldb, strideB, epi, M, N, K, batch)) return r;
  CUtensorMap tmA, tmB;
  int shareA, shareB, r;
  const int BN = N <= 64 ? 64 : 128;   // 64 accumulator registers per thread at most
  if ((r = make_operand_map(&tmA, A, a_mn, lda, strideA, M, K, batch, 128, &shareA))) return r;
  if ((r = make_operand_map(&tmB, B, b_mn, ldb, strideB, N, K, batch, BN, &shareB))) return r;
  if (BN == 64) return launch_gemm<64>(tmA, tmB, epi, M, N, K, batch, a_mn, b_mn, shareA, shareB, stream);
  return launch_gemm<128>(tmA, tmB, epi, M, N, K, batch, a_mn, b_mn, shareA, shareB, stream);
}

// C = epilogue(Ah.Bh + Al.Bh + Ah.Bl) in ONE launch; (Ah, Al) / (Bh, Bl) are tf32 (hi, lo) pairs with identical layouts.
int gemm_tf32_pair(const float* Ah, const float* Al, int a_mn, long long lda, long long strideA, const float* Bh,
                   const float* Bl, int b_mn, long long ldb, long long strideB, const GemmEpi& epi, int M, int N, int K,
                   int batch, cudaStream_t stream) {
  if (int r = check_gemm_args("gemm_pair", Ah, lda, strideA, Bh, ldb, strideB, epi, M, N, K, batch)) return r;
  if (int r = check_operand("gemm_pair", 'a', Al, lda, strideA, batch)) return r;
  if (int r = check_operand("gemm_pair", 'b', Bl, ldb, strideB, batch)) return r;
  CUtensorMap tmA, tmB, tmAl, tmBl;
  int shareA, shareB, r;
  // two accumulators per tile in registers: BN = 64 keeps them at 64 per thread
  const int BN = 64;
  if ((r = make_operand_map(&tmA, Ah, a_mn, lda, strideA, M, K, batch, 128, &shareA))) return r;
  if ((r = make_operand_map(&tmAl, Al, a_mn, lda, strideA, M, K, batch, 128, &shareA))) return r;
  if ((r = make_operand_map(&tmB, Bh, b_mn, ldb, strideB, N, K, batch, BN, &shareB))) return r;
  if ((r = make_operand_map(&tmBl, Bl, b_mn, ldb, strideB, N, K, batch, BN, &shareB))) return r;
  return launch_gemm<64>(tmA, tmB, epi, M, N, K, batch, a_mn, b_mn, shareA, shareB, stream, &tmAl, &tmBl);
}

__global__ void sum_splits_kernel(const float* __restrict__ part, int S, long long split_stride, long long ldp, int cols,
                                  size_t n, float* __restrict__ out, long long ldo, const float* __restrict__ bias,
                                  int accumulate) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / cols, c = i % cols;
    const float* p = part + r * ldp + c;
    float s = bias ? bias[c] : 0.f;
    for (int k = 0; k < S; ++k) s += p[(size_t)k * split_stride];
    float* o = out + r * ldo + c;
    *o = accumulate ? *o + s : s;
  }
}

int sum_splits(const float* part, int S, long long split_stride, int rows, int cols, long long ldp, float* out,
               long long ldo, const float* bias, bool accumulate, cudaStream_t stream) {
  const size_t n = (size_t)rows * cols;
  sum_splits_kernel<<<grid_1d(n, 256), 256, 0, stream>>>(part, S, split_stride, ldp, cols, n, out, ldo, bias,
                                                         accumulate ? 1 : 0);
  HK_LAUNCH_CHECK("sum_splits_kernel");
  return 0;
}

int gemm_splitk(const float* A, int a_mn, long long lda, const float* B, int b_mn, long long ldb, int M, int N, long long K,
                int S, float* part, float* out, long long ldo, int cols, const float* bias, bool accumulate,
                cudaStream_t stream) {
  const long long Kc = K / S;
  const bool direct = S == 1 && !bias && !accumulate && cols == N && ldo == N;
  GemmEpi e = {};
  e.C = direct ? out : part; e.ldc = N; e.strideC = (long long)M * N; e.alpha = 1.f;
  // batch index = K slice: slice s of a K-major operand starts s * Kc columns in, of an MN-major one s * Kc rows in
  int r = gemm_tf32(A, a_mn, lda, a_mn ? Kc * lda : Kc, B, b_mn, ldb, b_mn ? Kc * ldb : Kc, e, M, N, (int)Kc, S, stream);
  if (r || direct) return r;
  return sum_splits(part, S, (long long)M * N, M, cols, N, out, ldo, bias, accumulate, stream);
}

// the epilogue of hk_gemm_tf32 / hk_gemm_3xtf32 (see the public header)
static GemmEpi plain_epi(float* C, long long ldc, long long strideC, int trans_c, float alpha, const float* alpha_vec,
                         float diag, const float* D, long long ldd, long long strideD, float beta, const float* beta_vec,
                         int relu) {
  GemmEpi epi;
  epi.C = C; epi.ldc = ldc; epi.strideC = strideC;
  epi.D = D; epi.ldd = ldd; epi.strideD = strideD;
  epi.alpha_vec = alpha_vec; epi.beta_vec = beta_vec;
  epi.alpha = alpha; epi.beta = beta; epi.diag = diag;
  epi.trans_c = trans_c; epi.relu = relu;
  return epi;
}

}  // namespace hk

// same signature as hk_gemm_tf32, always 3xTF32 (callers whose result feeds an exponential: CIN's softmax(-Gram))
extern "C" int hk_gemm_3xtf32(const float* A, int a_mn_major, long long lda, long long strideA, const float* B,
                              int b_mn_major, long long ldb, long long strideB, float* C, long long ldc,
                              long long strideC, int trans_c, int M, int N, int K, int batch, float alpha,
                              const float* alpha_vec, float diag, const float* D, long long ldd, long long strideD,
                              float beta, const float* beta_vec, int relu, void* stream) {
  return hk::gemm_tf32_3x(A, a_mn_major, lda, strideA, B, b_mn_major, ldb, strideB,
                          hk::plain_epi(C, ldc, strideC, trans_c, alpha, alpha_vec, diag, D, ldd, strideD, beta, beta_vec, relu),
                          M, N, K, batch, static_cast<cudaStream_t>(stream));
}

extern "C" int hk_gemm_tf32(const float* A, int a_mn_major, long long lda, long long strideA, const float* B,
                            int b_mn_major, long long ldb, long long strideB, float* C, long long ldc,
                            long long strideC, int trans_c, int M, int N, int K, int batch, float alpha,
                            const float* alpha_vec, float diag, const float* D, long long ldd, long long strideD,
                            float beta, const float* beta_vec, int relu, void* stream) {
  return hk::gemm_tf32(A, a_mn_major, lda, strideA, B, b_mn_major, ldb, strideB,
                       hk::plain_epi(C, ldc, strideC, trans_c, alpha, alpha_vec, diag, D, ldd, strideD, beta, beta_vec, relu),
                       M, N, K, batch, static_cast<cudaStream_t>(stream));
}
