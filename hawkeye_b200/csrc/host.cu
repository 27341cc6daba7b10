// Error handling, version/introspection entry points and tensor-map construction.
#include "host.h"

#include <mutex>
#include <stdlib.h>
#include <string.h>

#include "../../include/hawkeye_b200.h"

namespace hk {

std::atomic<long long> g_launches{0};
static std::atomic<int> g_precise{-1};   // -1: not yet read from $HK_PRECISE

bool precise() {
  int v = g_precise.load();
  if (v < 0) {
    const char* e = getenv("HK_PRECISE");
    v = (e && atoi(e) != 0) ? 1 : 0;
    g_precise.store(v);
  }
  return v != 0;
}

int num_sms() {
  static const int sms = [] {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        n <= 0)
      return H100_SMS;
    return n;
  }();
  return sms;
}

Scratch::Scratch(size_t bytes, cudaStream_t stream) : s(stream) {
  if (cudaMallocAsync(&p, bytes ? bytes : 16, s) != cudaSuccess) { p = nullptr; (void)cudaGetLastError(); }
}
Scratch::~Scratch() {
  if (p) cudaFreeAsync(p, s);
}

char* last_error_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(last_error_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error(static_cast<int>(e), "%s: %s", what, cudaGetErrorString(e));
    return static_cast<int>(e);
  }
  return 0;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

int make_tmap(CUtensorMap* out, const float* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box, const uint32_t* elem_strides) {
  // the driver call needs a current context; autograd worker threads may not have bound one yet
  static thread_local bool ctx_ready = false;
  if (!ctx_ready) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, base) == cudaSuccess && at.type == cudaMemoryTypeDevice) cudaSetDevice(at.device);
    cudaFree(nullptr);
    (void)cudaGetLastError();
    ctx_ready = true;
  }
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(HK_ERR_DRIVER, "cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = elem_strides ? elem_strides[i] : 1;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    if (gstr[i] % 16 != 0)
      return set_error(HK_ERR_ALIGN, "tensor-map stride %d (%llu B) is not a multiple of 16", i,
                       (unsigned long long)gstr[i]);
  }
  if (!aligned16(base)) return set_error(HK_ERR_ALIGN, "tensor-map base pointer is not 16-byte aligned");
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, static_cast<cuuint32_t>(rank), const_cast<float*>(base),
                   gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(HK_ERR_DRIVER, "cuTensorMapEncodeTiled failed (CUresult %d; rank %d dims %llu,%llu box %u,%u)",
                     (int)r, rank, (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 0), bdim[0],
                     rank > 1 ? bdim[1] : 0);
  return 0;
}

}  // namespace hk

extern "C" {

const char* hk_version(void) { return "hawkeye_b200 0.1 (sm_90a; wgmma/TMA)"; }
const char* hk_last_error(void) { return hk::last_error_buf(); }
void hk_set_precise(int on) { hk::g_precise.store(on ? 1 : 0); }
int hk_get_precise(void) { return hk::precise() ? 1 : 0; }
long long hk_launch_count(void) { return hk::g_launches.load(); }
void hk_reset_launch_count(void) { hk::g_launches.store(0); }

}  // extern "C"
