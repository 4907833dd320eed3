// Shared host helpers (error reporting, TMA descriptor encoding) and small device conversions.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <string.h>

namespace uc {

// host ------------------------------------------------------------------------------------------
int set_error(int code, const char* fmt, ...);
int ensure_driver();
// rank-N tiled tensor map, 128B swizzle, zero OOB fill.  strides has rank-1 entries (bytes, dims 1..rank-1).
int encode_tmap(CUtensorMap* out, CUtensorMapDataType dt, int rank, const void* base, const uint64_t* dims,
                const uint64_t* strides, const uint32_t* box, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B);
int check_launch(const char* what);
int num_sms();
// One-time per-DEVICE state (cudaFuncSetAttribute, occupancy queries are per device): a process that drives several GPUs must not
// reuse what it cached for the first one.
constexpr int kMaxDevices = 64;
int cur_device();  // cudaGetDevice, clamped to [0, kMaxDevices)
struct PerDeviceFlag {
  bool done[kMaxDevices] = {};
  bool& get() { return done[cur_device()]; }
};
struct PerDeviceInt {
  int v[kMaxDevices] = {};
  int& get() { return v[cur_device()]; }
};
bool pdl_enabled();  // UC_PDL=0 in the environment turns programmatic dependent launch off (plain stream order)

// Launch with the programmatic-stream-serialization attribute: the kernel may become resident while its predecessor in
// the stream is still draining; every kernel launched this way calls pdl_wait() before it touches global memory.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

// GroupNorm statistics are accumulated as 64-bit fixed point (value * 2^22) with integer atomics so that the result
// does not depend on the order in which CTAs finish (bit-reproducible frames).
constexpr float kGnFixedScale = 4194304.f;

// device ----------------------------------------------------------------------------------------
#define UC_DT_BF16 0
#define UC_DT_F32 1
#define UC_DT_F16 2

__device__ __forceinline__ float bits16_to_float(uint32_t bits, int dtype) {
  if (dtype == UC_DT_F16) return __half2float(__ushort_as_half(static_cast<unsigned short>(bits)));
  return __uint_as_float(bits << 16);
}
__device__ __forceinline__ uint32_t float_to_bits16(float x, int dtype) {
  if (dtype == UC_DT_F16) return __half_as_ushort(__float2half_rn(x));
  return __bfloat16_as_ushort(__float2bfloat16_rn(x));
}
__device__ __forceinline__ uint32_t pack2_16(float lo, float hi, int dtype) {
  return float_to_bits16(lo, dtype) | (float_to_bits16(hi, dtype) << 16);
}
__device__ __forceinline__ float bf16lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  return __bfloat16_as_ushort(__float2bfloat16_rn(lo)) | (static_cast<uint32_t>(__bfloat16_as_ushort(__float2bfloat16_rn(hi))) << 16);
}

// acc += a * b on a pair of fp32 values packed in 64 bits (low word = first element)
__device__ __forceinline__ void fma_pair(unsigned long long& acc, unsigned long long a, unsigned long long b) {
  const float lo = fmaf(__uint_as_float(static_cast<uint32_t>(a)), __uint_as_float(static_cast<uint32_t>(b)), __uint_as_float(static_cast<uint32_t>(acc)));
  const float hi = fmaf(__uint_as_float(static_cast<uint32_t>(a >> 32)), __uint_as_float(static_cast<uint32_t>(b >> 32)),
                        __uint_as_float(static_cast<uint32_t>(acc >> 32)));
  acc = (static_cast<unsigned long long>(__float_as_uint(hi)) << 32) | __float_as_uint(lo);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace uc
