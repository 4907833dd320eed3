// Small data-movement kernels of the neck / embedding branch / prior pyramid (all HBM/L2-bound, vectorised).
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include <algorithm>

namespace uc {

// dst[b, oh, ow, :C] = src[b, oh/up, ow/up, :C]; 16-bit NHWC with pixel strides (dst may be a channel slice).
// yolo_pafpn_new.py:62,139-146 (nn.Upsample nearest x2 + torch.cat) when up == 2; plain slice copy when up == 1.
__global__ void __launch_bounds__(256) copy_upsample_kernel(const uint16_t* __restrict__ src, int lds, uint16_t* __restrict__ dst,
                                                             int ldd, int B, int Hs, int Ws, int C, int up) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int C8 = C >> 3;
  const int Hd = Hs * up, Wd = Ws * up;
  const long total = static_cast<long>(B) * Hd * Wd * C8;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(i % C8) * 8;
    long pix = i / C8;
    const int ow = static_cast<int>(pix % Wd);
    pix /= Wd;
    const int oh = static_cast<int>(pix % Hd);
    const int b = static_cast<int>(pix / Hd);
    const long sp = (static_cast<long>(b) * Hs + oh / up) * Ws + ow / up;
    const long dp = (static_cast<long>(b) * Hd + oh) * Wd + ow;
    *reinterpret_cast<uint4*>(dst + dp * ldd + c0) = __ldg(reinterpret_cast<const uint4*>(src + sp * lds + c0));
  }
}

// nn.PixelShuffle(2) in NHWC: in [B,H,W,4*Co] -> out [B,2H,2W,Co]; out[b,2h+i,2w+j,c] = in[b,h,w,c*4+i*2+j].
// unicorn.py:41.  16-bit elements; one thread per output (pixel, channel pair).
__global__ void __launch_bounds__(256) pixel_shuffle2_kernel(const uint16_t* __restrict__ in, int ldi, uint16_t* __restrict__ out,
                                                              int ldo, int B, int H, int W, int Co) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int Co2 = Co >> 1;
  const long total = static_cast<long>(B) * 2 * H * 2 * W * Co2;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % Co2) * 2;
    long pix = i / Co2;
    const int ow = static_cast<int>(pix % (2 * W));
    pix /= 2 * W;
    const int oh = static_cast<int>(pix % (2 * H));
    const int b = static_cast<int>(pix / (2 * H));
    const long sp = (static_cast<long>(b) * H + (oh >> 1)) * W + (ow >> 1);
    const int sub = (oh & 1) * 2 + (ow & 1);
    const uint32_t lo = in[sp * ldi + c * 4 + sub], hi = in[sp * ldi + (c + 1) * 4 + sub];
    const long dp = (static_cast<long>(b) * 2 * H + oh) * 2 * W + ow;
    *reinterpret_cast<uint32_t*>(out + dp * ldo + c) = lo | (hi << 16);
  }
}

// F.interpolate(mode="bilinear", align_corners=False) on fp32 planes [P,Hs,Ws] -> [P,Hd,Wd]
// (unicorn_sot.py:52-53,103-105; position_encoding.py:36).  PyTorch's source index rule:
// src = max(0, (dst + 0.5) * scale - 0.5), scale = Hs/Hd (or 1/scale_factor when a scale factor is given — equal here).
__global__ void __launch_bounds__(256) bilinear_kernel(const float* __restrict__ src, float* __restrict__ dst, int P, int Hs,
                                                        int Ws, int Hd, int Wd, float sh, float sw) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const long total = static_cast<long>(P) * Hd * Wd;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % Wd);
    const int y = static_cast<int>((i / Wd) % Hd);
    const int p = static_cast<int>(i / (static_cast<long>(Wd) * Hd));
    const float fy = fmaxf((y + 0.5f) * sh - 0.5f, 0.f), fx = fmaxf((x + 0.5f) * sw - 0.5f, 0.f);
    const int y0 = min(static_cast<int>(fy), Hs - 1), x0 = min(static_cast<int>(fx), Ws - 1);
    const int y1 = min(y0 + 1, Hs - 1), x1 = min(x0 + 1, Ws - 1);
    const float ly = fy - y0, lx = fx - x0;
    const float* s = src + static_cast<long>(p) * Hs * Ws;
    const float v = (1.f - ly) * ((1.f - lx) * s[y0 * Ws + x0] + lx * s[y0 * Ws + x1]) +
                    ly * ((1.f - lx) * s[y1 * Ws + x0] + lx * s[y1 * Ws + x1]);
    dst[i] = v;
  }
}

// ------------------------------------------------------------------------------------------------ letterbox (preprocessing)
// PreprocessorX.process (external/lib/test/tracker/unicorn_sot.py:114-123) / preproc (unicorn/data/data_augment.py:194-214):
// dst[0:rh, 0:rw] = cv2.resize(src, (rw, rh), INTER_LINEAR), everything else = pad (114), optionally RGB -> BGR.
// Bit-exact restatement of OpenCV's 8-bit bilinear (imgproc/resize.cpp: 11-bit fixed-point coefficients):
//   per axis  f = float((d + 0.5) * scale - 0.5), s = floor(f), f -= s, coefficients (short)rint((1-f)*2048), rint(f*2048);
//   x axis: s < 0 -> (s, f) = (0, 0); s >= W-1 -> (W-1, 0).  y axis: f is kept and the two source rows are clamped instead;
//   horizontal pass  h = S[sx]*a0 + S[sx+1]*a1 (int32);  vertical  (((b0*(h0>>4))>>16) + ((b1*(h1>>4))>>16) + 2) >> 2.
// One thread per output pixel (3 channels); the frame is read once from HBM (neighbouring threads share the source lines).
__device__ __forceinline__ void resize_axis(int d, double scale, int ssize, bool clamp, int& s0, int& s1, int& c0, int& c1) {
  float f = static_cast<float>((d + 0.5) * scale - 0.5);
  int s = static_cast<int>(floorf(f));
  f -= static_cast<float>(s);
  if (clamp) {
    if (s < 0) { s = 0; f = 0.f; }
    if (s >= ssize - 1) { s = ssize - 1; f = 0.f; }
  }
  c0 = __float2int_rn((1.f - f) * 2048.f);
  c1 = __float2int_rn(f * 2048.f);
  s0 = min(max(s, 0), ssize - 1);
  s1 = min(max(s + 1, 0), ssize - 1);
}

// Vertical pass of OpenCV's 8-bit bilinear on the horizontal sums h0 (row sy0) and h1 (row sy1).
__device__ __forceinline__ int resize_vert(int h0, int h1, int b0, int b1) {
  return (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
}

__global__ void __launch_bounds__(256) letterbox_u8_kernel(const uint8_t* __restrict__ src, int Hs, int Ws, uint8_t* __restrict__ dst, int Hd,
                                                            int Wd, int rh, int rw, double scale_y, double scale_x, int swap_rb, int pad) {
  pdl_wait();
  pdl_launch_dependents();
  const long total = static_cast<long>(Hd) * Wd;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % Wd), y = static_cast<int>(i / Wd);
    uint8_t o[3] = {static_cast<uint8_t>(pad), static_cast<uint8_t>(pad), static_cast<uint8_t>(pad)};
    if (x < rw && y < rh) {
      int sx0, sx1, a0, a1, sy0, sy1, b0, b1;
      resize_axis(x, scale_x, Ws, true, sx0, sx1, a0, a1);
      resize_axis(y, scale_y, Hs, false, sy0, sy1, b0, b1);
      const uint8_t* r0 = src + static_cast<long>(sy0) * Ws * 3;
      const uint8_t* r1 = src + static_cast<long>(sy1) * Ws * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int h0 = r0[sx0 * 3 + c] * a0 + r0[sx1 * 3 + c] * a1;
        const int h1 = r1[sx0 * 3 + c] * a0 + r1[sx1 * 3 + c] * a1;
        o[swap_rb ? 2 - c : c] = static_cast<uint8_t>(resize_vert(h0, h1, b0, b1));
      }
    }
    uint8_t* d = dst + i * 3;
    d[0] = o[0]; d[1] = o[1]; d[2] = o[2];
  }
}

// NV12 -> BGR as cv2.cvtColor(COLOR_YUV2BGR_NV12) computes it (OpenCV 4.x imgproc/src/color_yuv.simd.hpp: BT.601 limited range in
// 20-bit fixed point): Y' = max(0, Y - 16) * 1220542, u = U - 128, v = V - 128,
//   R = (Y' + 1673527 v + 2^19) >> 20,  G = (Y' - 852492 v - 409993 u + 2^19) >> 20,  B = (Y' + 2116026 u + 2^19) >> 20, each
// clamped to 0..255; chroma is nearest, the UV pair of pixel (r, c) is at row r >> 1, column c & ~1 of the interleaved plane.
__device__ __forceinline__ void nv12_bgr(const uint8_t* __restrict__ y, const uint8_t* __restrict__ uv, int ld, int r, int c, int bgr[3]) {
  const int yy = max(0, static_cast<int>(__ldg(y + static_cast<long>(r) * ld + c)) - 16) * 1220542;
  const uint8_t* p = uv + static_cast<long>(r >> 1) * ld + (c & ~1);
  const int u = static_cast<int>(__ldg(p)) - 128, v = static_cast<int>(__ldg(p + 1)) - 128;
  constexpr int half = 1 << 19;
  bgr[0] = min(max((yy + 2116026 * u + half) >> 20, 0), 255);
  bgr[1] = min(max((yy - 852492 * v - 409993 * u + half) >> 20, 0), 255);
  bgr[2] = min(max((yy + 1673527 * v + half) >> 20, 0), 255);
}

// letterbox_u8_kernel's output (swap_rb) for the BGR frame cv2.cvtColor(COLOR_YUV2BGR_NV12) makes of an NV12 frame: the four bilinear
// taps are converted to BGR in registers, so the BGR frame is never stored.  Y plane `y` and interleaved UV plane `uv` share the row
// pitch ld (bytes), so pitched decoder surfaces with padding rows between the planes are read in place.
__global__ void __launch_bounds__(256) letterbox_nv12_kernel(const uint8_t* __restrict__ y, const uint8_t* __restrict__ uv, int ld, int Hs,
                                                              int Ws, uint8_t* __restrict__ dst, int Hd, int Wd, int rh, int rw,
                                                              double scale_y, double scale_x, int pad) {
  pdl_wait();
  pdl_launch_dependents();
  const long total = static_cast<long>(Hd) * Wd;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % Wd), yo = static_cast<int>(i / Wd);
    uint8_t o[3] = {static_cast<uint8_t>(pad), static_cast<uint8_t>(pad), static_cast<uint8_t>(pad)};
    if (x < rw && yo < rh) {
      int sx0, sx1, a0, a1, sy0, sy1, b0, b1;
      resize_axis(x, scale_x, Ws, true, sx0, sx1, a0, a1);
      resize_axis(yo, scale_y, Hs, false, sy0, sy1, b0, b1);
      int p00[3], p01[3], p10[3], p11[3];
      nv12_bgr(y, uv, ld, sy0, sx0, p00);
      nv12_bgr(y, uv, ld, sy0, sx1, p01);
      nv12_bgr(y, uv, ld, sy1, sx0, p10);
      nv12_bgr(y, uv, ld, sy1, sx1, p11);
#pragma unroll
      for (int c = 0; c < 3; ++c)
        o[c] = static_cast<uint8_t>(resize_vert(p00[c] * a0 + p01[c] * a1, p10[c] * a0 + p11[c] * a1, b0, b1));
    }
    uint8_t* d = dst + i * 3;
    d[0] = o[0]; d[1] = o[1]; d[2] = o[2];
  }
}

// y = a + b (16-bit rows with strides), 8 elements per thread.
__global__ void __launch_bounds__(256) add_kernel(const uint16_t* __restrict__ a, int lda, const uint16_t* __restrict__ b, int ldb,
                                                   uint16_t* __restrict__ y, int ldy, long M, int C, int dtype) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int C8 = C >> 3;
  const long total = M * C8;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(i % C8) * 8;
    const long m = i / C8;
    const uint4 ua = __ldg(reinterpret_cast<const uint4*>(a + m * lda + c0));
    const uint4 ub = __ldg(reinterpret_cast<const uint4*>(b + m * ldb + c0));
    const uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w}, wb[4] = {ub.x, ub.y, ub.z, ub.w};
    uint32_t o[4];
#pragma unroll
    for (int t = 0; t < 4; ++t)
      o[t] = pack2_16(bits16_to_float(wa[t] & 0xffffu, dtype) + bits16_to_float(wb[t] & 0xffffu, dtype),
                      bits16_to_float(wa[t] >> 16, dtype) + bits16_to_float(wb[t] >> 16, dtype), dtype);
    *reinterpret_cast<uint4*>(y + m * ldy + c0) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// NCHW fp32 [B,C,H,W] -> NHWC 16-bit [B,H,W,C] and back (API boundary conversions; C % 2 == 0).
__global__ void __launch_bounds__(256) nchw_to_nhwc_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst, int ldd, int B,
                                                            int C, long HW, int dtype) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const long p0 = static_cast<long>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    const long p = p0 + tx;
    tile[j][tx] = (c < C && p < HW) ? src[(static_cast<long>(b) * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const long p = p0 + j;
    const int c = c0 + tx;
    if (p < HW && c < C) dst[(static_cast<long>(b) * HW + p) * ldd + c] = static_cast<uint16_t>(float_to_bits16(tile[tx][j], dtype));
  }
}
__global__ void __launch_bounds__(256) nhwc_to_nchw_kernel(const uint16_t* __restrict__ src, int lds, float* __restrict__ dst, int B,
                                                            int C, long HW, int dtype) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const long p0 = static_cast<long>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int j = ty; j < 32; j += 8) {
    const long p = p0 + j;
    const int c = c0 + tx;
    tile[j][tx] = (c < C && p < HW) ? bits16_to_float(src[(static_cast<long>(b) * HW + p) * lds + c], dtype) : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    const long p = p0 + tx;
    if (p < HW && c < C) dst[(static_cast<long>(b) * C + c) * HW + p] = tile[tx][j];
  }
}


// ------------------------------------------------------------------------------------------------ conditional row copy
// dst rows <- src rows when (*flag != 0) != invert, else nothing: device-side "pre_dict = cur_dict only if this frame had
// detections" (unicorn/evaluators/mot_evaluator.py:1005,1014-1020) without a host round trip, so the MOT frame stays one CUDA graph.
// blockIdx.y = image: image b copies src + b * src_bs to dst + b * dst_bs when (gate == NULL || gate[b] != 0) and
// (flag[b] != 0) != invert (a sequence slot that sits out a step keeps its pre_dict through the gate).
__global__ void __launch_bounds__(256) copy_rows_if_kernel(const int* __restrict__ flag, const int* __restrict__ gate, int invert,
                                                            const uint8_t* __restrict__ src, long src_ld, long src_bs, uint8_t* __restrict__ dst,
                                                            long dst_ld, long dst_bs, long rows, int row_chunks) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y;
  if ((gate && gate[b] == 0) || (flag[b] != 0) == (invert != 0)) return;
  src += b * src_bs;
  dst += b * dst_bs;
  const long total = rows * row_chunks;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long r = i / row_chunks;
    const int c = static_cast<int>(i % row_chunks);
    *reinterpret_cast<uint4*>(dst + r * dst_ld + c * 16) = *reinterpret_cast<const uint4*>(src + r * src_ld + c * 16);
  }
}

static inline int grid_for(long total, int per_block = 256) {
  return static_cast<int>(std::max<long>(1, std::min<long>((total + per_block - 1) / per_block, static_cast<long>(num_sms()) * 16)));
}

}  // namespace uc

using namespace uc;

extern "C" int uc_copy_upsample(const void* src, int lds, void* dst, int ldd, int B, int Hs, int Ws, int C, int up, void* stream_v) {
  if (!src || !dst || C % 8 || lds % 8 || ldd % 8 || (up != 1 && up != 2)) return set_error(UC_EINVAL, "uc_copy_upsample: bad arguments");
  if ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15)
    return set_error(UC_EINVAL, "uc_copy_upsample: src and dst must be 16-byte aligned");
  const long total = static_cast<long>(B) * Hs * up * Ws * up * (C / 8);
  launch_pdl(copy_upsample_kernel, grid_for(total), 256, 0, static_cast<cudaStream_t>(stream_v), 
      static_cast<const uint16_t*>(src), lds, static_cast<uint16_t*>(dst), ldd, B, Hs, Ws, C, up);
  return check_launch("uc_copy_upsample");
}

extern "C" int uc_pixel_shuffle2(const void* in, int ldi, void* out, int ldo, int B, int H, int W, int Co, void* stream_v) {
  if (!in || !out || Co % 2 || ldo % 2) return set_error(UC_EINVAL, "uc_pixel_shuffle2: bad arguments");
  const long total = static_cast<long>(B) * 4 * H * W * (Co / 2);
  launch_pdl(pixel_shuffle2_kernel, grid_for(total), 256, 0, static_cast<cudaStream_t>(stream_v), 
      static_cast<const uint16_t*>(in), ldi, static_cast<uint16_t*>(out), ldo, B, H, W, Co);
  return check_launch("uc_pixel_shuffle2");
}

extern "C" int uc_bilinear_f32(const float* src, float* dst, int P, int Hs, int Ws, int Hd, int Wd, float scale_h,
                               float scale_w, void* stream_v) {
  if (!src || !dst || P <= 0 || Hs <= 0 || Ws <= 0 || Hd <= 0 || Wd <= 0) return set_error(UC_EINVAL, "uc_bilinear_f32: bad arguments");
  const long total = static_cast<long>(P) * Hd * Wd;
  // scale_* = 1/scale_factor when the caller used F.interpolate(scale_factor=...), 0 -> size-based ratio
  launch_pdl(bilinear_kernel, grid_for(total), 256, 0, static_cast<cudaStream_t>(stream_v), 
      src, dst, P, Hs, Ws, Hd, Wd, scale_h > 0.f ? scale_h : static_cast<float>(Hs) / Hd,
      scale_w > 0.f ? scale_w : static_cast<float>(Ws) / Wd);
  return check_launch("uc_bilinear_f32");
}

extern "C" int uc_letterbox_u8(const uint8_t* src_hwc, int Hs, int Ws, uint8_t* dst_hwc, int Hd, int Wd, int rh, int rw, int swap_rb,
                               int pad, void* stream_v) {
  if (!src_hwc || !dst_hwc || Hs < 1 || Ws < 1 || Hd < 1 || Wd < 1 || rh < 1 || rw < 1 || rh > Hd || rw > Wd || pad < 0 || pad > 255)
    return set_error(UC_EINVAL, "uc_letterbox_u8: bad arguments");
  // cv::resize with an explicit dsize: inv_scale = dsize / ssize (double), scale = 1 / inv_scale
  const double scale_x = 1.0 / (static_cast<double>(rw) / Ws), scale_y = 1.0 / (static_cast<double>(rh) / Hs);
  launch_pdl(letterbox_u8_kernel, grid_for(static_cast<long>(Hd) * Wd), 256, 0, static_cast<cudaStream_t>(stream_v), src_hwc, Hs, Ws, dst_hwc,
             Hd, Wd, rh, rw, scale_y, scale_x, swap_rb, pad);
  return check_launch("uc_letterbox_u8");
}

extern "C" int uc_letterbox_nv12(const uint8_t* y, const uint8_t* uv, int ld, int Hs, int Ws, uint8_t* dst_hwc, int Hd, int Wd, int rh,
                                 int rw, int pad, void* stream_v) {
  if (!y || !uv || !dst_hwc) return set_error(UC_EINVAL, "uc_letterbox_nv12: null plane or destination");
  if (Hs < 2 || Ws < 2 || Hs % 2 || Ws % 2) return set_error(UC_EINVAL, "uc_letterbox_nv12: Hs and Ws must be even and >= 2");
  if (ld < Ws) return set_error(UC_EINVAL, "uc_letterbox_nv12: row pitch ld must be >= Ws");
  if (rh < 1 || rw < 1 || rh > Hd || rw > Wd) return set_error(UC_EINVAL, "uc_letterbox_nv12: rh, rw must be in 1..Hd, 1..Wd");
  if (pad < 0 || pad > 255) return set_error(UC_EINVAL, "uc_letterbox_nv12: pad must be in 0..255");
  const double scale_x = 1.0 / (static_cast<double>(rw) / Ws), scale_y = 1.0 / (static_cast<double>(rh) / Hs);
  launch_pdl(letterbox_nv12_kernel, grid_for(static_cast<long>(Hd) * Wd), 256, 0, static_cast<cudaStream_t>(stream_v), y, uv, ld, Hs, Ws,
             dst_hwc, Hd, Wd, rh, rw, scale_y, scale_x, pad);
  return check_launch("uc_letterbox_nv12");
}

extern "C" int uc_add(const void* a, int lda, const void* b, int ldb, void* y, int ldy, long M, int C, int dtype, void* stream_v) {
  if (!a || !b || !y || C % 8 || lda % 8 || ldb % 8 || ldy % 8) return set_error(UC_EINVAL, "uc_add: bad arguments");
  if (dtype != UC_BF16 && dtype != UC_F16) return set_error(UC_EINVAL, "uc_add: 16-bit dtypes only");
  if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(y)) & 15)
    return set_error(UC_EINVAL, "uc_add: a, b and y must be 16-byte aligned");
  launch_pdl(add_kernel, grid_for(M * (C / 8)), 256, 0, static_cast<cudaStream_t>(stream_v), 
      static_cast<const uint16_t*>(a), lda, static_cast<const uint16_t*>(b), ldb, static_cast<uint16_t*>(y), ldy, M, C, dtype);
  return check_launch("uc_add");
}

extern "C" int uc_nchw_f32_to_nhwc(const float* src, void* dst, int ldd, int B, int C, long HW, int dtype, void* stream_v) {
  if (!src || !dst || ldd < C) return set_error(UC_EINVAL, "uc_nchw_f32_to_nhwc: bad arguments");
  dim3 grid(static_cast<unsigned>((HW + 31) / 32), static_cast<unsigned>((C + 31) / 32), static_cast<unsigned>(B));
  launch_pdl(nchw_to_nhwc_kernel, grid, 256, 0, static_cast<cudaStream_t>(stream_v), src, static_cast<uint16_t*>(dst), ldd, B, C, HW, dtype);
  return check_launch("uc_nchw_f32_to_nhwc");
}

extern "C" int uc_nhwc_to_nchw_f32(const void* src, int lds, float* dst, int B, int C, long HW, int dtype, void* stream_v) {
  if (!src || !dst || lds < C) return set_error(UC_EINVAL, "uc_nhwc_to_nchw_f32: bad arguments");
  dim3 grid(static_cast<unsigned>((HW + 31) / 32), static_cast<unsigned>((C + 31) / 32), static_cast<unsigned>(B));
  launch_pdl(nhwc_to_nchw_kernel, grid, 256, 0, static_cast<cudaStream_t>(stream_v), static_cast<const uint16_t*>(src), lds, dst, B, C, HW, dtype);
  return check_launch("uc_nhwc_to_nchw_f32");
}

static int copy_rows_if(const char* name, const int* flag_dev, const int* gate_dev, int invert, const void* src, long src_ld_bytes,
                        long src_bs_bytes, void* dst, long dst_ld_bytes, long dst_bs_bytes, long rows, int row_bytes, int B, cudaStream_t stream) {
  launch_pdl(copy_rows_if_kernel, dim3(grid_for(rows * (row_bytes / 16)), B), 256, 0, stream, flag_dev, gate_dev, invert,
             static_cast<const uint8_t*>(src), src_ld_bytes, src_bs_bytes, static_cast<uint8_t*>(dst), dst_ld_bytes, dst_bs_bytes, rows,
             row_bytes / 16);
  return check_launch(name);
}

static bool aligned_rows(const void* src, long src_ld_bytes, const void* dst, long dst_ld_bytes, long rows, int row_bytes) {
  return rows >= 1 && row_bytes >= 16 && row_bytes % 16 == 0 && src_ld_bytes % 16 == 0 && dst_ld_bytes % 16 == 0 &&
         ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
}

extern "C" int uc_copy_rows_if(const int* flag_dev, int invert, const void* src, long src_ld_bytes, void* dst, long dst_ld_bytes, long rows,
                               int row_bytes, void* stream_v) {
  if (!flag_dev || !src || !dst || !aligned_rows(src, src_ld_bytes, dst, dst_ld_bytes, rows, row_bytes))
    return set_error(UC_EINVAL, "uc_copy_rows_if: 16-byte aligned rows only");
  return copy_rows_if("uc_copy_rows_if", flag_dev, nullptr, invert, src, src_ld_bytes, 0, dst, dst_ld_bytes, 0, rows, row_bytes, 1,
                      static_cast<cudaStream_t>(stream_v));
}

extern "C" int uc_copy_rows_if_batched(const int* flag_dev, const int* gate_dev, int invert, const void* src, long src_ld_bytes,
                                       long src_bs_bytes, void* dst, long dst_ld_bytes, long dst_bs_bytes, long rows, int row_bytes, int B,
                                       void* stream_v) {
  if (B < 1) return set_error(UC_EINVAL, "uc_copy_rows_if_batched: B must be >= 1");
  if (!flag_dev || !src || !dst) return set_error(UC_EINVAL, "uc_copy_rows_if_batched: null pointer");
  if (!aligned_rows(src, src_ld_bytes, dst, dst_ld_bytes, rows, row_bytes) || src_bs_bytes % 16 || dst_bs_bytes % 16)
    return set_error(UC_EINVAL, "uc_copy_rows_if_batched: 16-byte aligned rows only");
  if (src_bs_bytes < rows * src_ld_bytes || dst_bs_bytes < rows * dst_ld_bytes)
    return set_error(UC_EINVAL, "uc_copy_rows_if_batched: bad per-image strides (each must cover one image)");
  return copy_rows_if("uc_copy_rows_if_batched", flag_dev, gate_dev, invert, src, src_ld_bytes, src_bs_bytes, dst, dst_ld_bytes, dst_bs_bytes,
                      rows, row_bytes, B, static_cast<cudaStream_t>(stream_v));
}
