// Host-side helpers shared by the C-ABI translation units: error convention
// (0 ok / <0 argument error, no launch / >0 cudaError_t), thread-local last-error text,
// launch sizing (grid-stride grids, SM count, dynamic shared-memory opt-in)
// and CUtensorMap construction through the driver entry point (no libcuda link dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <atomic>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#define HK_OK 0
#define HK_ERR_ARG (-1)
#define HK_ERR_ALIGN (-2)
#define HK_ERR_UNSUPPORTED (-3)
#define HK_ERR_WORKSPACE (-4)
#define HK_ERR_DRIVER (-5)

namespace hk {

char* last_error_buf();
int set_error(int code, const char* fmt, ...);
int check_launch(const char* what);
extern std::atomic<long long> g_launches;  // kernels launched by this library (all host threads)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

constexpr int H100_SMS = 132;   // SMs of an H100 SXM

// Grid of a grid-stride kernel over n items: one thread per item, at least one block. The grid is capped at 16 blocks
// per SM: with 256-thread blocks that is two full waves (an SM holds 2048 threads), enough to keep every SM busy, and
// each thread's stride loop covers the remaining items more cheaply than further blocks would.
inline int grid_1d(size_t n, int block) {
  const size_t g = (n + block - 1) / block, cap = (size_t)H100_SMS * 16;
  return (int)(g < cap ? (g ? g : 1) : cap);
}

// SM count of the current device, looked up once per process (H100_SMS if the query fails).
int num_sms();

// Raise Kernel's dynamic shared-memory limit to `bytes` (above the 48 KB default). The attribute is set once per
// kernel: forward launches run on the caller's thread and backward launches on autograd's, and a function-local
// static is initialised exactly once even when both get here first at the same time. A failure is kept and returned
// on every call.
template <auto Kernel>
int allow_dynamic_smem(int bytes, const char* what) {
  static const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  return e == cudaSuccess ? 0 : set_error((int)e, "cudaFuncSetAttribute(%s): %s", what, cudaGetErrorString(e));
}

// Encode a tiled fp32 tensor map with SWIZZLE_128B and zero OOB fill.
// dims/box are innermost-first; strides_bytes[i] is the byte stride of dim i+1 (rank-1 entries).
int make_tmap(CUtensorMap* out, const float* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box, const uint32_t* elem_strides = nullptr);

// ---- precise mode (parity runs; hk_set_precise / $HK_PRECISE) -------------------------------------------------------
// 0 (default): every tensor-core product is single-pass TF32 and producers round what they hand to the next MMA.
// 1          : 3xTF32 — every MMA operand is split into (hi, lo) tf32 halves and A.B ~= Ah.Bh + Al.Bh + Ah.Bl is accumulated
//              by the same GEMM in one launch (its pair kernel issues all three products per k-step); nothing is rounded
//              on store.
//              fp32-class accuracy at >3x the cost: a test mode, which is why it may allocate stream-ordered scratch.
bool precise();
// stream-ordered scratch buffer (cudaMallocAsync / cudaFreeAsync on `s`); used by the precise mode only
struct Scratch {
  void* p = nullptr;
  cudaStream_t s;
  Scratch(size_t bytes, cudaStream_t stream);
  ~Scratch();
  float* f() const { return static_cast<float*>(p); }
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
};
// hi = rn_tf32(x), lo = rn_tf32(x - hi)  (elementwise over n floats; hi or lo may be null)
int tf32_split(const float* x, float* hi, float* lo, size_t n, cudaStream_t stream);

#define HK_REQUIRE(cond, code, ...) \
  do {                              \
    if (!(cond)) return hk::set_error(code, __VA_ARGS__); \
  } while (0)

#define HK_LAUNCH_CHECK(what)          \
  do {                                 \
    hk::g_launches++;                  \
    int _e = hk::check_launch(what);   \
    if (_e) return _e;                 \
  } while (0)

}  // namespace hk
