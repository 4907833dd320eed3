// ResNet-50 stem in one launch (unicorn/models/backbone/resnet.py:148-152,209-212):
//
//   conv1 7x7 stride 2 pad 3 (3 -> 64, BatchNorm folded into weights + bias) -> ReLU -> MaxPool2d(3, stride 2, pad 1)
//
// One CTA produces a kTPH x kTPW tile of the pooled map.  It needs the (2 kTPH + 1) x (2 kTPW + 1) conv pixels under the tile's
// pool windows (the extra top row / left column is the window overlap with the neighbouring tile, computed twice), which need a
// (2 CH + 5) x (2 CW + 5) input patch.  The patch is staged in shared memory as fp16; the conv is an implicit GEMM M = conv pixels,
// N = 64, K = 147 (padded to 160) on mma.sync m16n8k16 whose A fragments are gathered from the patch through a k -> offset table.
// Bias + ReLU are applied to the accumulators and the conv tile is written to shared memory as bf16 (rounding is monotonic, so
// max-pooling the rounded values equals rounding the max); the pool then reads it back and only the pooled map reaches HBM.
//
// Conv pixels outside the image are stored as 0: after the ReLU every value is >= 0 and every pool window holds at least one real
// pixel, so this equals the reference's -inf padding.
#include "uc_common.h"
#include "../../include/unicorn_b200.h"

namespace uc {

constexpr int kTPH = 8, kTPW = 16;                       // pooled tile
constexpr int kCH = 2 * kTPH + 1, kCW = 2 * kTPW + 1;    // conv tile 17 x 33
constexpr int kIH = 2 * kCH + 5, kIW = 2 * kCW + 5;      // input patch 39 x 71
constexpr int kStemM = kCH * kCW;                        // 561 conv pixels
constexpr int kStemMT = (kStemM + 15) / 16;              // 36 m16 tiles
constexpr int kStemK = 160;                              // 3 * 7 * 7 = 147 padded to 10 k16 steps
constexpr int kWLd = 168;                                // weight row stride (halves): conflict-free B fragment loads
constexpr int kStemThreads = 256;
constexpr int kInBytes = ((kIH * kIW * 3 * 2) + 127) / 128 * 128;
constexpr int kWBytes = 64 * kWLd * 2;
constexpr int kConvBytes = kStemM * 128;                 // bf16 [561][64], 16-byte chunks XOR-swizzled by (row & 7)
constexpr int kStemSmem = kInBytes + kWBytes + kConvBytes + kStemK * 4;

__device__ __forceinline__ void mma_f16_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(kStemThreads, 2) resnet_stem_kernel(const float* __restrict__ img, const uint8_t* __restrict__ img_u8,
                                                                      const __half* __restrict__ w, const float* __restrict__ bias,
                                                                      uint16_t* __restrict__ out, int H, int W) {
  extern __shared__ __align__(128) uint8_t smem[];
  __half* s_in = reinterpret_cast<__half*>(smem);                                   // [kIH][kIW][3]
  __half* s_w = reinterpret_cast<__half*>(smem + kInBytes);                         // [64][kWLd]
  uint8_t* s_conv = smem + kInBytes + kWBytes;                                      // [kStemM][8 chunks of 16 B]
  int* s_koff = reinterpret_cast<int*>(smem + kInBytes + kWBytes + kConvBytes);     // [160]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int b = blockIdx.z;
  const int Hc = H / 2, Wc = W / 2, Hp = H / 4, Wp = W / 4;
  const int py0 = blockIdx.y * kTPH, px0 = blockIdx.x * kTPW;
  const int cy0 = 2 * py0 - 1, cx0 = 2 * px0 - 1;   // conv tile origin
  const int iy0 = 2 * cy0 - 3, ix0 = 2 * cx0 - 3;   // input patch origin

  for (int i = tid; i < 64 * (kStemK / 8); i += kStemThreads) {
    const int n = i / (kStemK / 8), c = i % (kStemK / 8);
    *reinterpret_cast<uint4*>(s_w + n * kWLd + c * 8) = __ldg(reinterpret_cast<const uint4*>(w) + i);
  }
  for (int k = tid; k < kStemK; k += kStemThreads) {
    const int ci = k / 49, r = k % 49;
    s_koff[k] = k < 147 ? ((r / 7) * kIW + r % 7) * 3 + ci : 0;  // padded k: zero weight times any finite pixel
  }
  for (int i = tid; i < kIH * kIW * 3; i += kStemThreads) {
    const int ci = i % 3, c = (i / 3) % kIW, r = i / (3 * kIW);
    const int iy = iy0 + r, ix = ix0 + c;
    float v = 0.f;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
      v = img_u8 ? static_cast<float>(__ldg(img_u8 + ((static_cast<long>(b) * H + iy) * W + ix) * 3 + ci))
                 : __ldg(img + ((static_cast<long>(b) * 3 + ci) * H + iy) * W + ix);
    }
    s_in[i] = __float2half_rn(v);
  }
  __syncthreads();

  const uint16_t* in16 = reinterpret_cast<const uint16_t*>(s_in);
  for (int mt = warp; mt < kStemMT; mt += kStemThreads / 32) {
    int base[2];
    bool ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = min(mt * 16 + g + 8 * h, kStemM - 1);
      const int cy = row / kCW, cx = row % kCW;
      base[h] = (2 * cy * kIW + 2 * cx) * 3;
      const int gy = cy0 + cy, gx = cx0 + cx;
      ok[h] = gy >= 0 && gy < Hc && gx >= 0 && gx < Wc;
    }
    float acc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[nt][j] = 0.f;
#pragma unroll 2
    for (int ks = 0; ks < kStemK / 16; ++ks) {
      const int k0 = ks * 16 + 2 * t;
      const int o0 = s_koff[k0], o1 = s_koff[k0 + 1], o2 = s_koff[k0 + 8], o3 = s_koff[k0 + 9];
      const uint32_t a0 = in16[base[0] + o0] | (static_cast<uint32_t>(in16[base[0] + o1]) << 16);
      const uint32_t a1 = in16[base[1] + o0] | (static_cast<uint32_t>(in16[base[1] + o1]) << 16);
      const uint32_t a2 = in16[base[0] + o2] | (static_cast<uint32_t>(in16[base[0] + o3]) << 16);
      const uint32_t a3 = in16[base[1] + o2] | (static_cast<uint32_t>(in16[base[1] + o3]) << 16);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const __half* wp = s_w + (nt * 8 + g) * kWLd + k0;
        mma_f16_16816(acc[nt], a0, a1, a2, a3, *reinterpret_cast<const uint32_t*>(wp), *reinterpret_cast<const uint32_t*>(wp + 8));
      }
    }
    // bias + ReLU -> bf16 conv tile; accumulator (nt, j): row g + 8 (j >> 1), channel nt * 8 + 2 t + (j & 1)
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + nt * 8 + 2 * t));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = mt * 16 + g + 8 * h;
        if (row >= kStemM) continue;
        float v0 = acc[nt][2 * h] + bb.x, v1 = acc[nt][2 * h + 1] + bb.y;
        v0 = (ok[h] && v0 > 0.f) ? v0 : 0.f;  // +0 (never -0): the pool compares the bf16 bit patterns as unsigned integers
        v1 = (ok[h] && v1 > 0.f) ? v1 : 0.f;
        *reinterpret_cast<uint32_t*>(s_conv + row * 128 + ((nt ^ (row & 7)) << 4) + t * 4) = pack_bf16(v0, v1);
      }
    }
  }
  __syncthreads();

  // max-pool 3x3 stride 2: pooled (py, px) reads conv tile rows 2 (py - py0) + {0,1,2}, columns 2 (px - px0) + {0,1,2}
  for (int i = tid; i < kTPH * kTPW * 8; i += kStemThreads) {
    const int c8 = i & 7, pp = i >> 3;
    const int ply = pp / kTPW, plx = pp % kTPW;
    const int py = py0 + ply, px = px0 + plx;
    if (py >= Hp || px >= Wp) continue;
    uint4 m = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const int row = (2 * ply + dy) * kCW + 2 * plx + dx;
        const uint4 v = *reinterpret_cast<const uint4*>(s_conv + row * 128 + ((c8 ^ (row & 7)) << 4));
        m.x = __vmaxu2(m.x, v.x); m.y = __vmaxu2(m.y, v.y); m.z = __vmaxu2(m.z, v.z); m.w = __vmaxu2(m.w, v.w);
      }
    }
    *reinterpret_cast<uint4*>(out + ((static_cast<size_t>(b) * Hp + py) * Wp + px) * 64 + c8 * 8) = m;
  }
}

}  // namespace uc

using namespace uc;

extern "C" int uc_resnet_stem(const void* img, int img_is_u8_hwc, const void* w_f16, const float* bias, void* out_bf16, int B, int H, int W,
                              void* stream_v) {
  if (!img || !w_f16 || !bias || !out_bf16) return set_error(UC_EINVAL, "uc_resnet_stem: null pointer");
  if (B < 1 || H < 4 || W < 4 || H % 4 || W % 4) return set_error(UC_EINVAL, "uc_resnet_stem: need B >= 1, H %% 4 == 0, W %% 4 == 0 (H=%d W=%d)", H, W);
  if ((reinterpret_cast<uintptr_t>(w_f16) | reinterpret_cast<uintptr_t>(out_bf16)) & 15 || reinterpret_cast<uintptr_t>(bias) & 7)
    return set_error(UC_EINVAL, "uc_resnet_stem: w / out must be 16-byte and bias 8-byte aligned");
  static PerDeviceFlag attr_dev;
  bool& attr = attr_dev.get();
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(resnet_stem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kStemSmem);
    if (e != cudaSuccess) return set_error(static_cast<int>(e), "uc_resnet_stem: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr = true;
  }
  const dim3 grid((W / 4 + kTPW - 1) / kTPW, (H / 4 + kTPH - 1) / kTPH, B);
  resnet_stem_kernel<<<grid, kStemThreads, kStemSmem, static_cast<cudaStream_t>(stream_v)>>>(
      img_is_u8_hwc ? nullptr : static_cast<const float*>(img), img_is_u8_hwc ? static_cast<const uint8_t*>(img) : nullptr,
      static_cast<const __half*>(w_f16), bias, static_cast<uint16_t*>(out_bf16), H, W);
  return check_launch("uc_resnet_stem");
}
