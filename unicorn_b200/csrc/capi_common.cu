// Error reporting, device check and TMA descriptor encoding shared by every entry point.
#include <stdlib.h>
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include <stdarg.h>
#include <stdio.h>
#include <mutex>

namespace uc {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;
static std::once_flag g_once;
static int g_driver_rc = UC_EDRIVER;

int ensure_driver() {
  std::call_once(g_once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess && fn) {
      g_encode = reinterpret_cast<EncodeTiledFn>(fn);
      g_driver_rc = UC_OK;
    } else {
      cudaGetLastError();
    }
  });
  if (g_driver_rc) return set_error(UC_EDRIVER, "cuTensorMapEncodeTiled not available (no CUDA driver / GPU?)");
  return UC_OK;
}

int encode_tmap(CUtensorMap* out, CUtensorMapDataType dt, int rank, const void* base, const uint64_t* dims,
                const uint64_t* strides, const uint32_t* box, CUtensorMapSwizzle swz) {
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides[i];
  CUresult r = g_encode(out, dt, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gd, gs, bx, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return set_error(UC_EINVAL,
                     "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] strides [%llu %llu %llu] box [%u %u %u %u]",
                     static_cast<int>(r), rank, (unsigned long long)gd[0], (unsigned long long)(rank > 1 ? gd[1] : 0),
                     (unsigned long long)(rank > 2 ? gd[2] : 0), (unsigned long long)(rank > 3 ? gd[3] : 0),
                     (unsigned long long)gs[0], (unsigned long long)(rank > 2 ? gs[1] : 0),
                     (unsigned long long)(rank > 3 ? gs[2] : 0), bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0,
                     rank > 3 ? bx[3] : 0);
  }
  return UC_OK;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(static_cast<int>(e), "%s: %s", what, cudaGetErrorString(e));
  return UC_OK;
}

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("UC_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

int cur_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
  return dev < 0 ? 0 : (dev >= kMaxDevices ? kMaxDevices - 1 : dev);
}

int num_sms() {
  static PerDeviceInt cache;
  int& n = cache.get();
  if (!n) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, cur_device()) != cudaSuccess) {
      cudaGetLastError();
      n = 132;
    }
  }
  return n;
}

}  // namespace uc

extern "C" const char* uc_last_error(void) { return uc::g_err; }
extern "C" int uc_version(void) { return 100; }
extern "C" int uc_check_device(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) { cudaGetLastError(); return uc::set_error(UC_ENODEV, "no CUDA device: %s", cudaGetErrorString(e)); }
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) return uc::set_error(UC_ENODEV, "device compute capability %d.%d is not sm_90", major, minor);
  return uc::ensure_driver();
}
