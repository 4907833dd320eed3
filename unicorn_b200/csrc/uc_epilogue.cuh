// Epilogue arithmetic shared by the wgmma kernels (conv_gemm.cu, mlp_fused.cu): fp32 pairs, activations, 16-bit packing.
#pragma once
#include "uc_ptx.cuh"
#include "uc_common.h"
#include "../../include/unicorn_b200.h"

namespace uc {

__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// ---- fp32 pairs: the epilogues work on the (even, odd) column pairs a thread holds in a wgmma accumulator
typedef float2 f32x2;
__device__ __forceinline__ f32x2 pk2(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ float lo2(f32x2 v) { return v.x; }
__device__ __forceinline__ float hi2(f32x2 v) { return v.y; }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float fast_rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// exact (erf) GELU, nn.GELU(), as x * sigmoid(x * P(x^2)): P is the degree-4 least-squares fit of logit(Phi(x)) / x,
// max |error| 3.3e-6 over the whole real line (tools/fit_gelu.py; the bf16 output ulp is >= 1.5e-5 wherever |y| > 4e-3,
// and the fit saturates correctly: y -> x for x -> +inf, y -> -0 for x -> -inf).  Per element: 8 FMA-pipe instructions
// + (ex2, rcp), about a third of the issue slots of an Abramowitz-Stegun erf.
__device__ __forceinline__ f32x2 gelu2(f32x2 x) {
  // coefficients pre-multiplied by -log2(e): e = 2^(x * P'(x^2)) = exp(-q(x))
  const f32x2 c0 = pk2(-2.30204844f, -2.30204844f), c1 = pk2(-0.105217814f, -0.105217814f), c2 = pk2(3.54831049e-4f, 3.54831049e-4f),
              c3 = pk2(8.93110919e-5f, 8.93110919e-5f), c4 = pk2(-3.29185241e-6f, -3.29185241e-6f), one = pk2(1.f, 1.f);
  const f32x2 t = mul2(x, x);
  f32x2 pz = fma2(c4, t, c3);
  pz = fma2(pz, t, c2);
  pz = fma2(pz, t, c1);
  pz = fma2(pz, t, c0);
  const f32x2 u = mul2(x, pz);
  const f32x2 d = add2(pk2(fast_ex2(lo2(u)), fast_ex2(hi2(u))), one);
  return mul2(x, pk2(fast_rcp(lo2(d)), fast_rcp(hi2(d))));
}
__device__ __forceinline__ float gelu_erf(float x) { return lo2(gelu2(pk2(x, x))); }
__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case UC_ACT_RELU: return fmaxf(x, 0.f);
    case UC_ACT_GELU: return gelu_erf(x);
    case UC_ACT_SILU: return x * fast_rcp(1.f + fast_ex2(-x * 1.4426950408889634f));
    case UC_ACT_SIGMOID: return fast_rcp(1.f + fast_ex2(-x * 1.4426950408889634f));
    default: return x;
  }
}
__device__ __forceinline__ uint32_t pack2_fast(float lo, float hi, bool f16) {  // one F2FP per pair
  if (f16) { const __half2 h = __floats2half2_rn(lo, hi); return *reinterpret_cast<const uint32_t*>(&h); }
  const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

}  // namespace uc
