// HBM/L2-bound CUDA-core kernels of the backbone: stem conv4x4s4+LN, depthwise 7x7 + LayerNorm, LayerNorm,
// GroupNorm apply (+SiLU / prior fusion).  All activations NHWC; statistics and arithmetic in fp32.
#include "uc_common.h"
#include "../../include/unicorn_b200.h"

namespace uc {

// ------------------------------------------------------------------------------------------------ stem
// convnext.py:77-80: Conv2d(3, C0, k=4, s=4) + LayerNorm(channels_first, eps 1e-6).
// img fp32 NCHW [B,3,H,W]; w packed [48][C0] fp32 (k = (ci*4+kh)*4+kw); out NHWC bf16 [B,H/4,W/4,C0].
// One warp handles 4 horizontally adjacent output pixels; lane owns channels lane+32*i.
template <int CPL>  // channels per lane = C0/32
__global__ void __launch_bounds__(256) stem_ln_kernel(const float* __restrict__ img, const uint8_t* __restrict__ img_u8, const float* __restrict__ w,
                                                       const float* __restrict__ bias, const float* __restrict__ lnw,
                                                       const float* __restrict__ lnb, uint16_t* __restrict__ out, int B,
                                                       int H, int W, float eps) {
  extern __shared__ float sw[];  // [48][C0]
  const int C0 = CPL * 32;
  for (int i = threadIdx.x; i < 48 * C0; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int Ho = H / 4, Wo = W / 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int groups_w = (Wo + 3) / 4;
  const long total = static_cast<long>(B) * Ho * groups_w;
  for (long g = static_cast<long>(blockIdx.x) * 8 + warp; g < total; g += static_cast<long>(gridDim.x) * 8) {
    const int gw = static_cast<int>(g % groups_w);
    const int oh = static_cast<int>((g / groups_w) % Ho);
    const int b = static_cast<int>(g / (static_cast<long>(groups_w) * Ho));
    const int ow0 = gw * 4;
    // lanes 0..47 each fetch one (ci,kh) row segment of 16 contiguous floats? simpler: each lane loads inputs
    // k = lane and k = lane+32 (k<48) for the 4 pixels -> shuffle-broadcast in the FMA loop.
    float in0[4], in1[4];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int ow = ow0 + p;
      {
        const int k = lane, ci = k >> 4, kh = (k >> 2) & 3, kw = k & 3;
        if (ow >= Wo) in0[p] = 0.f;
        else if (img_u8) in0[p] = static_cast<float>(__ldg(img_u8 + ((static_cast<long>(b) * H + oh * 4 + kh) * W + ow * 4 + kw) * 3 + ci));
        else in0[p] = __ldg(img + ((static_cast<long>(b) * 3 + ci) * H + oh * 4 + kh) * W + ow * 4 + kw);
      }
      {
        const int k = lane + 32;
        if (k < 48) {
          const int ci = k >> 4, kh = (k >> 2) & 3, kw = k & 3;
          if (ow >= Wo) in1[p] = 0.f;
          else if (img_u8) in1[p] = static_cast<float>(__ldg(img_u8 + ((static_cast<long>(b) * H + oh * 4 + kh) * W + ow * 4 + kw) * 3 + ci));
          else in1[p] = __ldg(img + ((static_cast<long>(b) * 3 + ci) * H + oh * 4 + kh) * W + ow * 4 + kw);
        } else {
          in1[p] = 0.f;
        }
      }
    }
    float acc[4][CPL];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int i = 0; i < CPL; ++i) acc[p][i] = __ldg(bias + lane + 32 * i);
#pragma unroll 8
    for (int k = 0; k < 48; ++k) {
      float xv[4];
#pragma unroll
      for (int p = 0; p < 4; ++p) xv[p] = __shfl_sync(0xffffffffu, k < 32 ? in0[p] : in1[p], k & 31);
#pragma unroll
      for (int i = 0; i < CPL; ++i) {
        const float wv = sw[k * C0 + lane + 32 * i];
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[p][i] = fmaf(xv[p], wv, acc[p][i]);
      }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < CPL; ++i) s += acc[p][i];
      const float mean = warp_sum(s) / C0;
      float v = 0.f;
#pragma unroll
      for (int i = 0; i < CPL; ++i) { const float d = acc[p][i] - mean; v += d * d; }
      const float rstd = rsqrtf(warp_sum(v) / C0 + eps);
      const int ow = ow0 + p;
      if (ow < Wo) {
        uint16_t* o = out + ((static_cast<long>(b) * Ho + oh) * Wo + ow) * C0;
#pragma unroll
        for (int i = 0; i < CPL; ++i) {
          const int c = lane + 32 * i;
          o[c] = static_cast<uint16_t>(float_to_bits16((acc[p][i] - mean) * rstd * __ldg(lnw + c) + __ldg(lnb + c), UC_DT_BF16));
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ dwconv7 + LN
// convnext.py:43-45: depthwise 7x7 (pad 3, bias) -> LayerNorm over C (eps 1e-6).  x NHWC bf16 -> y NHWC bf16.
// w packed [49][C] fp32.  Block = one row segment of PX pixels x all C channels; thread = one channel pair.
constexpr int kDwPx = 8;
__global__ void __launch_bounds__(768) dwconv7_ln_kernel(const uint32_t* __restrict__ x, const float2* __restrict__ w,
                                                          const float2* __restrict__ bias, const float2* __restrict__ lnw,
                                                          const float2* __restrict__ lnb, uint32_t* __restrict__ y, int B,
                                                          int H, int W, int C2 /* C/2 */, float eps) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  __shared__ float red[2][kDwPx][32];
  const int segs = (W + kDwPx - 1) / kDwPx;
  const int seg = blockIdx.x % segs;
  const int oh = (blockIdx.x / segs) % H;
  const int b = blockIdx.x / (segs * H);
  const int ow0 = seg * kDwPx;
  const int cp = threadIdx.x;  // channel pair
  const bool active = cp < C2;
  float a0[kDwPx], a1[kDwPx];
  if (active) {
    const float2 bb = __ldg(bias + cp);
#pragma unroll
    for (int p = 0; p < kDwPx; ++p) { a0[p] = bb.x; a1[p] = bb.y; }
#pragma unroll 1
    for (int kh = 0; kh < 7; ++kh) {
      const int ih = oh + kh - 3;
      if (ih < 0 || ih >= H) continue;
      const uint32_t* row = x + (static_cast<long>(b) * H + ih) * W * C2 + cp;
      float v0[kDwPx + 6], v1[kDwPx + 6];
#pragma unroll
      for (int j = 0; j < kDwPx + 6; ++j) {
        const int iw = ow0 + j - 3;
        uint32_t u = 0;
        if (iw >= 0 && iw < W) u = __ldg(row + static_cast<long>(iw) * C2);
        v0[j] = bf16lo(u); v1[j] = bf16hi(u);
      }
#pragma unroll
      for (int kw = 0; kw < 7; ++kw) {
        const float2 wv = __ldg(w + (kh * 7 + kw) * C2 + cp);
#pragma unroll
        for (int p = 0; p < kDwPx; ++p) {
          a0[p] = fmaf(v0[p + kw], wv.x, a0[p]);
          a1[p] = fmaf(v1[p + kw], wv.y, a1[p]);
        }
      }
    }
  } else {
#pragma unroll
    for (int p = 0; p < kDwPx; ++p) { a0[p] = 0.f; a1[p] = 0.f; }
  }
  // LayerNorm over channels: two-pass block reduction per pixel
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  float mean[kDwPx], rstd[kDwPx];
#pragma unroll
  for (int p = 0; p < kDwPx; ++p) {
    const float s = warp_sum(a0[p] + a1[p]);
    if (lane == 0) red[0][p][warp] = s;
  }
  __syncthreads();
#pragma unroll
  for (int p = 0; p < kDwPx; ++p) {
    float s = 0.f;
    for (int i = 0; i < nwarps; ++i) s += red[0][p][i];
    mean[p] = s / (2 * C2);
  }
#pragma unroll
  for (int p = 0; p < kDwPx; ++p) {
    const float d0 = a0[p] - mean[p], d1 = a1[p] - mean[p];
    const float s = warp_sum(active ? d0 * d0 + d1 * d1 : 0.f);
    if (lane == 0) red[1][p][warp] = s;
  }
  __syncthreads();
#pragma unroll
  for (int p = 0; p < kDwPx; ++p) {
    float s = 0.f;
    for (int i = 0; i < nwarps; ++i) s += red[1][p][i];
    rstd[p] = rsqrtf(s / (2 * C2) + eps);
  }
  if (active) {
    const float2 gw = __ldg(lnw + cp), gb = __ldg(lnb + cp);
#pragma unroll
    for (int p = 0; p < kDwPx; ++p) {
      const int ow = ow0 + p;
      if (ow < W) {
        y[((static_cast<long>(b) * H + oh) * W + ow) * C2 + cp] =
            pack_bf16((a0[p] - mean[p]) * rstd[p] * gw.x + gb.x, (a1[p] - mean[p]) * rstd[p] * gw.y + gb.y);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ dwconv7 + LayerNorm (fused)
// ConvNeXt block head (convnext.py:43-45, 48): y = LN_C(dwconv7x7(x) + bias).  One CTA owns a TW x TH pixel tile and ALL C
// channels of it: it walks the channels in chunks of 64, staging each chunk's (TW+6) x (TH+6) halo tile and its 49 x 64
// filter taps with cp.async (double buffered: chunk k+1 streams in while chunk k is computed), computes the depthwise
// outputs as channel-pair FMAs (fma_pair) and parks them as bf16 in a [pixels][C] shared-memory buffer; a second phase
// does the (two-pass, fp32) LayerNorm of every pixel from that buffer and writes full 128-byte lines.  The intermediate
// map never exists in global memory and the two launches of the unfused path (uc_dwconv7 + uc_layernorm) become one.
// The rounding points are the same as the unfused path (conv output rounded to bf16 before the LayerNorm).
template <int TW, int TH, int PX, int NT>
__global__ void __launch_bounds__(NT) dwln_kernel(const uint16_t* __restrict__ x, const float* __restrict__ w,
                                                   const float* __restrict__ bias, const float* __restrict__ lnw,
                                                   const float* __restrict__ lnb, uint16_t* __restrict__ y, int H, int W, int C,
                                                   int tiles_w, float eps) {
  constexpr int CCH = 64, PAIRS = 32, HW_ = TW + 6, HH_ = TH + 6, PIX_BYTES = CCH * 2, P = TW * TH, GW = TW / PX;
  static_assert(GW * TH * PAIRS == NT, "one thread per (channel pair, PX-pixel group)");
  constexpr int HALO_BYTES = HH_ * HW_ * PIX_BYTES, W_BYTES = 49 * CCH * 4;
  extern __shared__ __align__(16) uint8_t dsm[];
  uint32_t* outb = reinterpret_cast<uint32_t*>(dsm + 2 * HALO_BYTES + 2 * W_BYTES);  // [P][C/2] bf16 pairs
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y;
  const int ow0 = (blockIdx.x % tiles_w) * TW, oh0 = (blockIdx.x / tiles_w) * TH;
  const uint16_t* xb = x + static_cast<long>(b) * H * W * C;
  const int C2 = C >> 1, nchunks = C / CCH;

  auto load_chunk = [&](int k, int buf) {
    uint8_t* tile = dsm + buf * HALO_BYTES;
    uint8_t* swb = dsm + 2 * HALO_BYTES + buf * W_BYTES;
    const int c0 = k * CCH;
    for (int i = threadIdx.x; i < HH_ * HW_ * 8; i += NT) {
      const int ch = i & 7, px = i >> 3;
      const int hx = px % HW_, hy = px / HW_;
      const int ih = oh0 + hy - 3, iw = ow0 + hx - 3;
      uint8_t* dst = tile + px * PIX_BYTES + ch * 16;
      if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
        const uint16_t* src = xb + (static_cast<long>(ih) * W + iw) * C + c0 + ch * 8;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))), "l"(src) : "memory");
      } else {
        *reinterpret_cast<uint4*>(dst) = make_uint4(0u, 0u, 0u, 0u);
      }
    }
    for (int i = threadIdx.x; i < 49 * 16; i += NT) {
      const int tap = i >> 4, u = i & 15;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(swb + tap * 256 + u * 16))),
                   "l"(w + static_cast<long>(tap) * C + c0 + u * 4)
                   : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  const int cp = threadIdx.x % PAIRS;
  const int grp = threadIdx.x / PAIRS;
  const int gx = grp % GW, r = grp / GW;
  load_chunk(0, 0);
#pragma unroll 1
  for (int k = 0; k < nchunks; ++k) {
    const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + k * CCH) + cp);
    if (k + 1 < nchunks) {
      load_chunk(k + 1, (k + 1) & 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const uint8_t* tile = dsm + (k & 1) * HALO_BYTES;
    const float* sw = reinterpret_cast<const float*>(dsm + 2 * HALO_BYTES + (k & 1) * W_BYTES);
    unsigned long long acc[PX];
    {
      const unsigned long long bb = (static_cast<unsigned long long>(__float_as_uint(bv.y)) << 32) | __float_as_uint(bv.x);
#pragma unroll
      for (int p = 0; p < PX; ++p) acc[p] = bb;
    }
#pragma unroll 1
    for (int kh = 0; kh < 7; ++kh) {
      const uint32_t* rowp = reinterpret_cast<const uint32_t*>(tile + ((r + kh) * HW_ + gx * PX) * PIX_BYTES) + cp;
      unsigned long long v[PX + 6];
#pragma unroll
      for (int j = 0; j < PX + 6; ++j) {
        const uint32_t u = rowp[j * (PIX_BYTES / 4)];
        v[j] = (static_cast<unsigned long long>(u & 0xffff0000u) << 32) | (u << 16);  // (lo -> .x, hi -> .y) as fp32 bits
      }
#pragma unroll
      for (int kw = 0; kw < 7; ++kw) {
        const unsigned long long wv = *reinterpret_cast<const unsigned long long*>(sw + (kh * 7 + kw) * CCH + 2 * cp);
#pragma unroll
        for (int p = 0; p < PX; ++p) fma_pair(acc[p], v[p + kw], wv);
      }
    }
#pragma unroll
    for (int p = 0; p < PX; ++p) {
      outb[(r * TW + gx * PX + p) * C2 + k * PAIRS + cp] =
          pack_bf16(__uint_as_float(static_cast<uint32_t>(acc[p] & 0xffffffffull)), __uint_as_float(static_cast<uint32_t>(acc[p] >> 32)));
    }
    __syncthreads();  // chunk k's buffers may be refilled (iteration k+1 prefetches chunk k+2 into them)
  }
  // ---- LayerNorm over the channels of every pixel of the tile: one warp per pixel, two-pass statistics in fp32
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float inv_c = 1.f / static_cast<float>(C);
  for (int px = warp; px < P; px += NT / 32) {
    const int ow = ow0 + px % TW, oh = oh0 + px / TW;
    if (ow >= W || oh >= H) continue;
    const uint32_t* row = outb + px * C2;
    float s = 0.f;
    for (int c = lane; c < C2; c += 32) { const uint32_t u = row[c]; s += bf16lo(u) + bf16hi(u); }
    const float mean = warp_sum(s) * inv_c;
    float qv = 0.f;
    for (int c = lane; c < C2; c += 32) {
      const uint32_t u = row[c];
      const float d0 = bf16lo(u) - mean, d1 = bf16hi(u) - mean;
      qv = fmaf(d0, d0, qv);
      qv = fmaf(d1, d1, qv);
    }
    const float rstd = rsqrtf(warp_sum(qv) * inv_c + eps);
    uint32_t* yr = reinterpret_cast<uint32_t*>(y + ((static_cast<long>(b) * H + oh) * W + ow) * C);
    for (int c = lane; c < C2; c += 32) {
      const uint32_t u = row[c];
      const float2 gw = __ldg(reinterpret_cast<const float2*>(lnw) + c), gb = __ldg(reinterpret_cast<const float2*>(lnb) + c);
      yr[c] = pack_bf16((bf16lo(u) - mean) * rstd * gw.x + gb.x, (bf16hi(u) - mean) * rstd * gw.y + gb.y);
    }
  }
}

template <int TW, int TH, int PX, int NT>
static bool launch_dwln(const void* x, const float* w49, const float* bias, const float* lnw, const float* lnb, void* y, int B, int H,
                        int W, int C, float eps, cudaStream_t stream, bool force) {
  constexpr int smem_fixed = 2 * (TH + 6) * (TW + 6) * 128 + 2 * 49 * 64 * 4;
  const int smem = smem_fixed + TW * TH * C * 2;
  const int tiles_w = (W + TW - 1) / TW, tiles = tiles_w * ((H + TH - 1) / TH);
  if (smem > 227 * 1024) return false;
  if (!force && static_cast<long>(tiles) * B < 100) return false;  // too few CTAs for the SMs: try a smaller tile
  static PerDeviceInt smem_dev;
  int& smem_set = smem_dev.get();
  auto kern = dwln_kernel<TW, TH, PX, NT>;
  if (smem > smem_set) { cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); smem_set = smem; }
  launch_pdl(kern, dim3(tiles, B), NT, smem, stream, static_cast<const uint16_t*>(x), w49, bias, lnw, lnb, static_cast<uint16_t*>(y), H, W, C,
             tiles_w, eps);
  return true;
}

// ------------------------------------------------------------------------------------------------ LayerNorm rows
// y[m, :] = LN(x[m, :] (+ r[m, :])) * w + b, one warp per row, C <= 2048, C even.  x/r/y 16-bit rows with strides.
template <int MAXI>  // bf16 pairs per lane: C <= 64 * MAXI
__global__ void __launch_bounds__(256) layernorm_kernel(const uint16_t* __restrict__ x, int ldx,
                                                         const uint16_t* __restrict__ r, int ldr,
                                                         const float* __restrict__ w, const float* __restrict__ bvec,
                                                         uint16_t* __restrict__ y, int ldy, long M, int C, float eps,
                                                         int dtype) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int lane = threadIdx.x & 31;
  const long m = static_cast<long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (m >= M) return;
  float v0[MAXI], v1[MAXI];
  const uint32_t* xr = reinterpret_cast<const uint32_t*>(x + m * ldx);
  const uint32_t* rr = r ? reinterpret_cast<const uint32_t*>(r + m * ldr) : nullptr;
  const int C2 = C >> 1;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    const int c = lane + 32 * i;
    v0[i] = 0.f; v1[i] = 0.f;
    if (c < C2) {
      const uint32_t u = __ldg(xr + c);
      v0[i] = bits16_to_float(u & 0xffffu, dtype); v1[i] = bits16_to_float(u >> 16, dtype);
      if (rr) {
        const uint32_t u2 = __ldg(rr + c);
        v0[i] += bits16_to_float(u2 & 0xffffu, dtype); v1[i] += bits16_to_float(u2 >> 16, dtype);
      }
      s += v0[i] + v1[i];
    }
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    if (lane + 32 * i < C2) { const float d0 = v0[i] - mean, d1 = v1[i] - mean; q += d0 * d0 + d1 * d1; }
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  uint32_t* yr = reinterpret_cast<uint32_t*>(y + m * ldy);
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    const int c = lane + 32 * i;
    if (c < C2) {
      const float2 ww = __ldg(reinterpret_cast<const float2*>(w) + c), bb = __ldg(reinterpret_cast<const float2*>(bvec) + c);
      yr[c] = pack2_16((v0[i] - mean) * rstd * ww.x + bb.x, (v1[i] - mean) * rstd * ww.y + bb.y, dtype);
    }
  }
}

// Same LayerNorm with 128-bit accesses: a lane owns 8-channel chunks lane + 32 i (C % 8 == 0, 16-byte aligned rows); the affine
// parameters of the first chunks are requested before the two warp reductions so that their latency is hidden behind them.
template <int MAXV>  // 8-channel chunks per lane: C <= 256 * MAXV
__global__ void __launch_bounds__(256) layernorm_v8_kernel(const uint16_t* __restrict__ x, int ldx, const uint16_t* __restrict__ r, int ldr,
                                                            const float* __restrict__ w, const float* __restrict__ bvec,
                                                            uint16_t* __restrict__ y, int ldy, long M, int C, float eps, int dtype) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const long m = static_cast<long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (m >= M) return;
  const int C8 = C >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + m * ldx);
  const uint4* rr = r ? reinterpret_cast<const uint4*>(r + m * ldr) : nullptr;
  float v[MAXV][8];
  constexpr int PRE = MAXV <= 3 ? MAXV : 0;  // chunks whose gamma / beta are prefetched (register budget)
  float4 gw[PRE > 0 ? PRE : 1][2], gb[PRE > 0 ? PRE : 1][2];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = lane + 32 * i;
#pragma unroll
    for (int j = 0; j < 8; ++j) v[i][j] = 0.f;
    if (c < C8) {
      const uint4 u = __ldg(xr + c);
      const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) { v[i][2 * t] = bits16_to_float(uw[t] & 0xffffu, dtype); v[i][2 * t + 1] = bits16_to_float(uw[t] >> 16, dtype); }
      if (rr) {
        const uint4 u2 = __ldg(rr + c);
        const uint32_t rw[4] = {u2.x, u2.y, u2.z, u2.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) { v[i][2 * t] += bits16_to_float(rw[t] & 0xffffu, dtype); v[i][2 * t + 1] += bits16_to_float(rw[t] >> 16, dtype); }
      }
      if (i < PRE) {
        gw[i][0] = __ldg(reinterpret_cast<const float4*>(w) + 2 * c); gw[i][1] = __ldg(reinterpret_cast<const float4*>(w) + 2 * c + 1);
        gb[i][0] = __ldg(reinterpret_cast<const float4*>(bvec) + 2 * c); gb[i][1] = __ldg(reinterpret_cast<const float4*>(bvec) + 2 * c + 1);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    }
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    if (lane + 32 * i < C8) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; q = fmaf(d, d, q); }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  uint4* yr = reinterpret_cast<uint4*>(y + m * ldy);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = lane + 32 * i;
    if (c < C8) {
      float4 w0, w1, b0, b1;
      if (i < PRE) { w0 = gw[i][0]; w1 = gw[i][1]; b0 = gb[i][0]; b1 = gb[i][1]; }
      else {
        w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * c); w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * c + 1);
        b0 = __ldg(reinterpret_cast<const float4*>(bvec) + 2 * c); b1 = __ldg(reinterpret_cast<const float4*>(bvec) + 2 * c + 1);
      }
      const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w}, bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * ww[j] + bb[j];
      uint4 u;
      u.x = pack2_16(o[0], o[1], dtype); u.y = pack2_16(o[2], o[3], dtype); u.z = pack2_16(o[4], o[5], dtype); u.w = pack2_16(o[6], o[7], dtype);
      yr[c] = u;
    }
  }
}

// ------------------------------------------------------------------------------------------------ GroupNorm apply
// y = act(x * scale[c] + shift[c]) (+ prior[pix] * beta[c]); optional second output y2 = y + add2.
// scale/shift fold the group statistics (int64 fixed point {sum, sumsq} accumulated by uc_conv2d) with the affine
// parameters; they are computed once per block into shared memory.  x/y bf16 NHWC (strided); 8 channels / thread.
// kMode says which image of x and of the statistics output image b (blockIdx.y) reads:
//   kGnEach    image b (uc_groupnorm_apply);
//   kGnGather  image src_of[b] of the n_src images of x, read once per CTA; only the images b >= prior_from add the prior, reading
//              its plane b - prior_from; the others take the no-prior path.  An entry outside [0, n_src) leaves image b untouched.
//              y2 is unused.
enum GnApplyMode { kGnEach, kGnGather };
template <int kMode>
__global__ void __launch_bounds__(256) groupnorm_apply_kernel(const uint16_t* __restrict__ x, int ldx,
                                                               const long long* __restrict__ stats, const float* __restrict__ w,
                                                               const float* __restrict__ bvec, uint16_t* __restrict__ y, int ldy,
                                                               long HW, int C, int G, float eps, int act,
                                                               const float* __restrict__ prior, const float* __restrict__ beta,
                                                               const uint16_t* __restrict__ add2, int ldadd2,
                                                               uint16_t* __restrict__ y2, int ldy2, int prior_from,
                                                               const int* __restrict__ src_of, int n_src) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  extern __shared__ float sc[];  // [2][C] scale, shift (+ [C] beta)
  const int b = blockIdx.y;
  const int bx = kMode == kGnEach ? b : src_of[b];  // image of x and of the statistics
  if (kMode == kGnGather && (bx < 0 || bx >= n_src)) return;  // uniform over the CTA, before any barrier
  const bool with_prior = prior != nullptr && (kMode == kGnEach || b >= prior_from);
  const int gs = C / G;
  const double inv_n = 1.0 / (static_cast<double>(HW) * gs);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / gs;
    const double sum = static_cast<double>(stats[(static_cast<long>(bx) * G + g) * 2]) * (1.0 / kGnFixedScale);
    const double sq = static_cast<double>(stats[(static_cast<long>(bx) * G + g) * 2 + 1]) * (1.0 / kGnFixedScale);
    const double mean = sum * inv_n;
    const float var = fmaxf(static_cast<float>(sq * inv_n - mean * mean), 0.f);
    const float rstd = rsqrtf(var + eps);
    const float a = rstd * w[c];
    sc[c] = a;
    sc[C + c] = bvec[c] - static_cast<float>(mean) * a;
    sc[2 * C + c] = beta ? beta[c] : 0.f;
  }
  __syncthreads();
  const int C8 = C >> 3;
  const long total = HW * C8;
  const bool silu = act == UC_ACT_SILU, relu = act == UC_ACT_RELU;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(i % C8) * 8;
    const long pix = static_cast<long>(b) * HW + i / C8;
    const long xpix = kMode == kGnEach ? pix : static_cast<long>(bx) * HW + i / C8;
    const uint4 u = *reinterpret_cast<const uint4*>(x + xpix * ldx + c0);
    const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
    // per-channel coefficients as 128-bit shared-memory loads (c0 is a multiple of 8 -> 32-byte aligned)
    const float4 s0 = *reinterpret_cast<const float4*>(sc + c0), s1 = *reinterpret_cast<const float4*>(sc + c0 + 4);
    const float4 h0 = *reinterpret_cast<const float4*>(sc + C + c0), h1 = *reinterpret_cast<const float4*>(sc + C + c0 + 4);
    const float scl[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float sft[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
    float f[8];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      f[2 * t] = fmaf(bf16lo(uw[t]), scl[2 * t], sft[2 * t]);
      f[2 * t + 1] = fmaf(bf16hi(uw[t]), scl[2 * t + 1], sft[2 * t + 1]);
    }
    if (silu) {  // x * sigmoid(x) with ex2.approx / rcp.approx (~1 ulp each; the result is rounded to bf16)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float e, r;
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-f[j] * 1.4426950408889634f));
        asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.f + e));
        f[j] *= r;
      }
    } else if (relu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaxf(f[j], 0.f);
    }
    if (with_prior) {
      const float pr = __ldg(prior + (kMode != kGnEach ? static_cast<long>(b - prior_from) * HW + i / C8 : pix));
      const float4 b0 = *reinterpret_cast<const float4*>(sc + 2 * C + c0), b1 = *reinterpret_cast<const float4*>(sc + 2 * C + c0 + 4);
      const float bt[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaf(pr, bt[j], f[j]);
    }
    uint4 o;
    o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]); o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
    *reinterpret_cast<uint4*>(y + pix * ldy + c0) = o;
    if (kMode == kGnEach && y2) {
      const uint4 a = *reinterpret_cast<const uint4*>(add2 + pix * ldadd2 + c0);
      const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
      uint4 o2;
      o2.x = pack_bf16(f[0] + bf16lo(aw[0]), f[1] + bf16hi(aw[0]));
      o2.y = pack_bf16(f[2] + bf16lo(aw[1]), f[3] + bf16hi(aw[1]));
      o2.z = pack_bf16(f[4] + bf16lo(aw[2]), f[5] + bf16hi(aw[2]));
      o2.w = pack_bf16(f[6] + bf16lo(aw[3]), f[7] + bf16hi(aw[3]));
      *reinterpret_cast<uint4*>(y2 + pix * ldy2 + c0) = o2;
    }
  }
}

}  // namespace uc

using namespace uc;

extern "C" int uc_stem_ln(const void* img, int img_is_u8_hwc, const float* w48, const float* bias, const float* lnw, const float* lnb,
                          void* out_bf16, int B, int H, int W, int C0, float eps, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!img || !w48 || !bias || !lnw || !lnb || !out_bf16) return set_error(UC_EINVAL, "uc_stem_ln: null pointer");
  if (H % 4 || W % 4 || C0 % 32 || C0 > 256) return set_error(UC_EINVAL, "uc_stem_ln: need H%%4==0, W%%4==0, C0%%32==0, C0<=256");
  const long groups = static_cast<long>(B) * (H / 4) * ((W / 4 + 3) / 4);
  const int grid = static_cast<int>(std::min<long>((groups + 7) / 8, static_cast<long>(num_sms()) * 8));
  const size_t smem = static_cast<size_t>(48) * C0 * sizeof(float);
  uint16_t* out = static_cast<uint16_t*>(out_bf16);
#define UC_STEM(CPL)                                                                                                   \
  case CPL: {                                                                                                          \
    cudaFuncSetAttribute(stem_ln_kernel<CPL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);                 \
    stem_ln_kernel<CPL><<<grid, 256, smem, stream>>>(img_is_u8_hwc ? nullptr : static_cast<const float*>(img),                  \
                                                     img_is_u8_hwc ? static_cast<const uint8_t*>(img) : nullptr, w48, bias, lnw, lnb, out, B, H, W, eps);                     \
  } break;
  switch (C0 / 32) {
    UC_STEM(1) UC_STEM(2) UC_STEM(3) UC_STEM(4) UC_STEM(6) UC_STEM(8)
    default: return set_error(UC_EINVAL, "uc_stem_ln: unsupported C0 %d", C0);
  }
#undef UC_STEM
  return check_launch("uc_stem_ln");
}

extern "C" int uc_dwconv7_ln(const void* x_bf16, const float* w49, const float* bias, const float* lnw, const float* lnb,
                             void* y_bf16, int B, int H, int W, int C, float eps, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!x_bf16 || !w49 || !bias || !lnw || !lnb || !y_bf16) return set_error(UC_EINVAL, "uc_dwconv7_ln: null pointer");
  if (x_bf16 == y_bf16) return set_error(UC_EINVAL, "uc_dwconv7_ln: not an in-place operation");
  if (C % 2 || C > 1536 || C < 2) return set_error(UC_EINVAL, "uc_dwconv7_ln: C must be even and <= 1536");
  if (C % 64 == 0) {
    // largest pixel tile that still gives every SM a CTA and fits its [pixels][C] buffer in shared memory
    bool ok = launch_dwln<16, 8, 8, 512>(x_bf16, w49, bias, lnw, lnb, y_bf16, B, H, W, C, eps, stream, false) ||
              launch_dwln<8, 8, 8, 256>(x_bf16, w49, bias, lnw, lnb, y_bf16, B, H, W, C, eps, stream, false) ||
              launch_dwln<8, 4, 4, 256>(x_bf16, w49, bias, lnw, lnb, y_bf16, B, H, W, C, eps, stream, false) ||
              launch_dwln<4, 2, 1, 256>(x_bf16, w49, bias, lnw, lnb, y_bf16, B, H, W, C, eps, stream, true);
    if (!ok) return set_error(UC_EINVAL, "uc_dwconv7_ln: no tile configuration fits (C=%d)", C);
    return check_launch("uc_dwconv7_ln");
  }
  const int C2 = C / 2;
  const int threads = (C2 + 31) / 32 * 32;
  const long blocks = static_cast<long>(B) * H * ((W + kDwPx - 1) / kDwPx);
  if (blocks > 0x7fffffffL) return set_error(UC_EINVAL, "uc_dwconv7_ln: too many blocks");
  launch_pdl(dwconv7_ln_kernel, static_cast<unsigned>(blocks), threads, 0, stream, 
      static_cast<const uint32_t*>(x_bf16), reinterpret_cast<const float2*>(w49), reinterpret_cast<const float2*>(bias),
      reinterpret_cast<const float2*>(lnw), reinterpret_cast<const float2*>(lnb), static_cast<uint32_t*>(y_bf16), B, H, W, C2, eps);
  return check_launch("uc_dwconv7_ln");
}

extern "C" int uc_layernorm(const void* x, int ldx, const void* res, int ldres, const float* w, const float* b, void* y,
                            int ldy, long M, int C, float eps, int dtype, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!x || !w || !b || !y) return set_error(UC_EINVAL, "uc_layernorm: null pointer");
  if (C % 2 || C > 2048 || ldx % 2 || ldy % 2 || (res && ldres % 2)) return set_error(UC_EINVAL, "uc_layernorm: C even <= 2048, even strides");
  if (dtype != UC_BF16 && dtype != UC_F16) return set_error(UC_EINVAL, "uc_layernorm: 16-bit dtypes only");
  const long blocks = (M + 7) / 8;
  const bool v8 = C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && (!res || ldres % 8 == 0) &&
                  ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(res)) & 15) == 0;
  if (v8) {
#define UC_LNV(MAXV)                                                                                                     \
  launch_pdl(layernorm_v8_kernel<MAXV>, static_cast<unsigned>(blocks), 256, 0, stream,                                          \
      static_cast<const uint16_t*>(x), ldx, static_cast<const uint16_t*>(res), ldres, w, b, static_cast<uint16_t*>(y), ldy, M, C, eps, dtype)
    if (C <= 256) UC_LNV(1);
    else if (C <= 512) UC_LNV(2);
    else if (C <= 768) UC_LNV(3);
    else if (C <= 1536) UC_LNV(6);
    else UC_LNV(8);
#undef UC_LNV
    return check_launch("uc_layernorm");
  }
#define UC_LN(MAXI)                                                                                                      \
  launch_pdl(layernorm_kernel<MAXI>, static_cast<unsigned>(blocks), 256, 0, stream,                                             \
      static_cast<const uint16_t*>(x), ldx, static_cast<const uint16_t*>(res), ldres, w, b, static_cast<uint16_t*>(y), ldy, M, C, eps, dtype)
  if (C <= 128) UC_LN(2);
  else if (C <= 256) UC_LN(4);
  else if (C <= 384) UC_LN(6);
  else if (C <= 768) UC_LN(12);
  else if (C <= 1536) UC_LN(24);
  else UC_LN(32);
#undef UC_LN
  return check_launch("uc_layernorm");
}

extern "C" int uc_groupnorm_apply(const void* x, int ldx, const void* stats, const float* w, const float* b, void* y,
                                  int ldy, int B, long HW, int C, int G, float eps, int act, const float* prior,
                                  const float* beta, const void* add2, int ldadd2, void* y2, int ldy2, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  // sizes before pointers: G is checked before it divides anything
  if (G < 1) return set_error(UC_EINVAL, "uc_groupnorm_apply: G must be >= 1 (got %d)", G);
  if (C % 8 || ldx % 8 || ldy % 8 || C % G) return set_error(UC_EINVAL, "uc_groupnorm_apply: C, ldx, ldy multiples of 8; C %% G == 0");
  if (C > 4096) return set_error(UC_EINVAL, "uc_groupnorm_apply: C too large");
  if (act != UC_ACT_NONE && act != UC_ACT_RELU && act != UC_ACT_SILU)
    return set_error(UC_EINVAL, "uc_groupnorm_apply: act must be UC_ACT_NONE, UC_ACT_RELU or UC_ACT_SILU (got %d)", act);
  if (!x || !stats || !w || !b || !y) return set_error(UC_EINVAL, "uc_groupnorm_apply: null pointer");
  if ((prior != nullptr) != (beta != nullptr)) return set_error(UC_EINVAL, "uc_groupnorm_apply: prior and beta go together");
  if (y2 && (!add2 || ldadd2 % 8 || ldy2 % 8)) return set_error(UC_EINVAL, "uc_groupnorm_apply: bad second output");
  // the kernel moves 8 channels per 128-bit access
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(add2) | reinterpret_cast<uintptr_t>(y2)) & 15)
    return set_error(UC_EINVAL, "uc_groupnorm_apply: x, y, add2 and y2 must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(stats) & 7) return set_error(UC_EINVAL, "uc_groupnorm_apply: stats must be 8-byte aligned");
  const long total = HW * (C / 8);
  // each block pays C scale/shift computations up front; keep ~2 elements (16 channels) per thread for parallelism
  const int gx = static_cast<int>(std::max<long>(1, std::min<long>((total + 256 * 2 - 1) / (256 * 2), static_cast<long>(num_sms()) * 8)));
  launch_pdl(groupnorm_apply_kernel<kGnEach>, dim3(gx, B), 256, 3 * C * sizeof(float), stream,
      static_cast<const uint16_t*>(x), ldx, reinterpret_cast<const long long*>(stats), w, b, static_cast<uint16_t*>(y), ldy, HW, C, G,
      eps, act, prior, beta, static_cast<const uint16_t*>(add2), ldadd2, static_cast<uint16_t*>(y2), ldy2, 0,
      static_cast<const int*>(nullptr), 0);
  return check_launch("uc_groupnorm_apply");
}

extern "C" int uc_groupnorm_apply_gather(const void* x, int ldx, int n_src, const void* stats, const float* w, const float* b, void* y,
                                         int ldy, int B, int n_plain, const int* src_of, long HW, int C, int G, float eps, int act,
                                         const float* prior, const float* beta, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_src < 1 || n_src > 65535) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: n_src must be in [1, 65535] (got %d)", n_src);
  if (B < 1 || B > 65535) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: B must be in [1, 65535] (got %d)", B);
  if (n_plain < 0 || n_plain > B) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: n_plain must be in [0, B] (got %d, B = %d)", n_plain, B);
  if (HW < 1) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: HW must be >= 1");
  if (G < 1) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: G must be >= 1 (got %d)", G);
  if (C % 8 || ldx % 8 || ldy % 8 || C % G || ldx < C || ldy < C)
    return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: C, ldx, ldy multiples of 8, ldx, ldy >= C; C %% G == 0");
  if (C > 4096) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: C too large");
  if (act != UC_ACT_NONE && act != UC_ACT_RELU && act != UC_ACT_SILU)
    return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: act must be UC_ACT_NONE, UC_ACT_RELU or UC_ACT_SILU (got %d)", act);
  if (!x || !stats || !w || !b || !y || !src_of) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: null pointer");
  if ((prior != nullptr) != (beta != nullptr)) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: prior and beta go together");
  if ((prior != nullptr) != (n_plain < B))
    return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: prior and beta are needed exactly when n_plain < B");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15)
    return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: x and y must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(stats) & 7) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: stats must be 8-byte aligned");
  if (reinterpret_cast<uintptr_t>(prior) & 3) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: prior must be 4-byte aligned");
  if (reinterpret_cast<uintptr_t>(src_of) & 3) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: src_of must be 4-byte aligned");
  // an output image may read any of the n_src images: writing any of them over x would race with the other images' reads
  const uintptr_t x0 = reinterpret_cast<uintptr_t>(x), y0 = reinterpret_cast<uintptr_t>(y);
  const uintptr_t x1 = x0 + (static_cast<uintptr_t>(n_src) * HW - 1) * ldx * 2 + static_cast<uintptr_t>(C) * 2;  // one past the last element
  const uintptr_t y1 = y0 + (static_cast<uintptr_t>(B) * HW - 1) * ldy * 2 + static_cast<uintptr_t>(C) * 2;
  if (x0 < y1 && y0 < x1) return set_error(UC_EINVAL, "uc_groupnorm_apply_gather: x and y overlap (not an in-place operation)");
  const long total = HW * (C / 8);
  const int gx = static_cast<int>(std::max<long>(1, std::min<long>((total + 256 * 2 - 1) / (256 * 2), static_cast<long>(num_sms()) * 8)));
  launch_pdl(groupnorm_apply_kernel<kGnGather>, dim3(gx, B), 256, 3 * C * sizeof(float), stream,
      static_cast<const uint16_t*>(x), ldx, reinterpret_cast<const long long*>(stats), w, b, static_cast<uint16_t*>(y), ldy, HW, C, G,
      eps, act, prior, beta, static_cast<const uint16_t*>(nullptr), 0, static_cast<uint16_t*>(nullptr), 0, n_plain, src_of, n_src);
  return check_launch("uc_groupnorm_apply_gather");
}
