// Depthwise 7x7 convolution (pad 3) + bias of the ConvNeXt block (unicorn/models/backbone/convnext.py:43, :21), TMA staged.
//
//   y[b, oh, ow, c] = bias[c] + sum_{kh,kw} x[b, oh+kh-3, ow+kw-3, c] * w[kh*7+kw][c]          x, y NHWC bf16, w fp32 [49][C]
//
// Work item = a 16 x 8 output tile of one 64-channel chunk.  ONE elected thread asks the TMA engine for the item's
// (16+6) x (8+6) x 64-channel input box — a 4-D box {64 ch, 22, 14, 1} of the NHWC map whose out-of-map part (the zero padding
// of the convolution, negative coordinates included) is zero-filled by the hardware — and for the chunk's 49 x 64 fp32 filter
// taps; both land in one of TWO shared-memory stages and complete on that stage's mbarrier, so the box of item n+1 streams in
// while item n is computed.  No thread computes an address or a bounds check for the staging.
//
// The kernel is bound by fp32 FMA issue, not by HBM (98 flop per output element, 15.6 GFLOP per 800x1280 frame), and register
// blocking keeps the shared-memory reads per FMA low: 256 threads = 8 warps; a warp owns an 8-pixel strip of TWO output rows, a lane
// one channel pair; per staged input row (14 pixels, read and converted once) it issues 2 x 56 channel-pair FMAs (fma_pair) — with
// filter row kh for the upper output row and the previous filter row, kept in registers, for the lower one.  Items are handed out by
// an atomic counter (a static split gives uneven per-SM loads on small maps).
//
// Optional per-pixel LayerNorm statistics (sum, sum of squares over C of the STORED bf16 values, int64 fixed point 2^22, integer
// atomics: order independent) feed the following pwconv1, which applies the normalisation in its epilogue (UcConv2d.row_stats).
#include "uc_ptx.cuh"
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include <algorithm>

namespace uc {

constexpr int kDwTW = 16, kDwTH = 8, kDwCCH = 64, kDwPX = 8, kDwR = 2;
constexpr int kDwHW = kDwTW + 6, kDwHH = kDwTH + 6;               // 22 x 14 input box
constexpr int kDwPixBytes = kDwCCH * 2;                             // 128 B per staged pixel
constexpr int kDwTileBytes = kDwHH * kDwHW * kDwPixBytes;           // 39424
constexpr int kDwWBytes = 49 * kDwCCH * 4;                          // 12544
constexpr int kDwStageBytes = kDwTileBytes + kDwWBytes;             // 51968 (multiple of 128)
constexpr int kDwThreads = (kDwTW / kDwPX) * (kDwTH / kDwR) * 32;   // 256
constexpr int kDwSmem = 2 * kDwStageBytes + 128 + 128;              // two stages + barriers / item slots + alignment slack
constexpr int kDwCtasPerSm = 2;

struct alignas(64) DwParams {
  CUtensorMap tmX, tmW;
  const float* bias;
  uint16_t* y;
  unsigned long long* ln_stats;
  int* work_counter;  // zeroed by the caller; nullptr = static round-robin
  int H, W, C, B, tiles_w, tiles_h, n_items;
};

__global__ void __launch_bounds__(kDwThreads, kDwCtasPerSm) dwconv7_tma_kernel(const __grid_constant__ DwParams p) {
  extern __shared__ uint8_t dsm_raw[];
  uint8_t* base = dsm_raw + ((128u - (smem_u32(dsm_raw) & 127u)) & 127u);  // 128-byte aligned; the pointer stays a shared-memory pointer (LDS, not LD)
  uint64_t* bar = reinterpret_cast<uint64_t*>(base + 2 * kDwStageBytes);    // full[2]
  volatile int* s_item = reinterpret_cast<volatile int*>(bar + 2);          // item index staged per stage (-1 = no more work)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int hx = warp & 1, rp = warp >> 1;  // this warp's strip: pixels 8 hx .. 8 hx + 7 of tile rows 2 rp, 2 rp + 1
  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tmX);
    prefetch_tmap(&p.tmW);
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();
  const int tiles_img = p.tiles_w * p.tiles_h, tiles_chunk = tiles_img * p.B;
  const int C2 = p.C >> 1;
  int static_next = blockIdx.x;  // thread 0 only

  // thread 0: claim items (the atomic's round trip is hidden: an index is consumed one iteration after it was requested) and start
  // the loads of an item into `stage` (the stage's previous readers are behind a __syncthreads)
  auto fetch = [&]() {
    if (p.work_counter) return atomicAdd(p.work_counter, 1);
    const int item = static_next;
    static_next += gridDim.x;
    return item;
  };
  auto issue = [&](int stage, int item) {
    if (item >= p.n_items) {
      s_item[stage] = -1;
      mbar_arrive(&bar[stage]);
      return;
    }
    s_item[stage] = item;
    const int chunk = item / tiles_chunk, t = item - chunk * tiles_chunk;
    const int b = t / tiles_img, tt = t - b * tiles_img;
    const int oh0 = (tt / p.tiles_w) * kDwTH, ow0 = (tt % p.tiles_w) * kDwTW;
    uint8_t* dst = base + stage * kDwStageBytes;
    mbar_arrive_expect_tx(&bar[stage], kDwStageBytes);
    tma_load_4d(dst, &p.tmX, &bar[stage], chunk * kDwCCH, ow0 - 3, oh0 - 3, b);
    tma_load_2d(dst + kDwTileBytes, &p.tmW, &bar[stage], chunk * kDwCCH, 0);
  };
  int pending = 0;
  if (threadIdx.x == 0) {
    issue(0, fetch());
    pending = fetch();
  }
  for (int it = 0;; ++it) {
    const int stage = it & 1;
    if (threadIdx.x == 0) {
      issue(stage ^ 1, pending);
      pending = fetch();
    }
    mbar_wait(&bar[stage], (it >> 1) & 1);
    const int item = s_item[stage];
    if (item < 0) break;
    const uint8_t* tile = base + stage * kDwStageBytes;                          // [14][22][64] bf16
    const float* sw = reinterpret_cast<const float*>(tile + kDwTileBytes);      // [49][64] fp32
    const int chunk = item / tiles_chunk, t = item - chunk * tiles_chunk;
    const int b = t / tiles_img, tt = t - b * tiles_img;
    const int oh0 = (tt / p.tiles_w) * kDwTH, ow0 = (tt % p.tiles_w) * kDwTW;
    const int c = chunk * kDwCCH + 2 * lane;  // this lane's channel pair (C is even: both channels are in range or neither)
    const bool c_ok = c < p.C;
    unsigned long long acc[kDwR][kDwPX];
    {
      const float2 bv = c_ok ? __ldg(reinterpret_cast<const float2*>(p.bias + c)) : make_float2(0.f, 0.f);
      const unsigned long long bb = (static_cast<unsigned long long>(__float_as_uint(bv.y)) << 32) | __float_as_uint(bv.x);
#pragma unroll
      for (int r = 0; r < kDwR; ++r)
#pragma unroll
        for (int q = 0; q < kDwPX; ++q) acc[r][q] = bb;
    }
    unsigned long long wprev[7];
#pragma unroll
    for (int i = 0; i < 8; ++i) {  // input row 2 rp + i of the box: filter row i for output row 2 rp, filter row i - 1 for 2 rp + 1
      const uint32_t* rowp = reinterpret_cast<const uint32_t*>(tile + ((kDwR * rp + i) * kDwHW + hx * kDwPX) * kDwPixBytes) + lane;
      unsigned long long v[kDwPX + 6];
#pragma unroll
      for (int j = 0; j < kDwPX + 6; ++j) {
        const uint32_t u = rowp[j * (kDwPixBytes / 4)];
        v[j] = (static_cast<unsigned long long>(u & 0xffff0000u) << 32) | (u << 16);  // (lo -> .x, hi -> .y) as fp32 bits
      }
      unsigned long long wcur[7];
      if (i < 7) {
#pragma unroll
        for (int kw = 0; kw < 7; ++kw) wcur[kw] = *reinterpret_cast<const unsigned long long*>(sw + (i * 7 + kw) * kDwCCH + 2 * lane);
#pragma unroll
        for (int kw = 0; kw < 7; ++kw)
#pragma unroll
          for (int q = 0; q < kDwPX; ++q) fma_pair(acc[0][q], v[q + kw], wcur[kw]);
      }
      if (i > 0) {
#pragma unroll
        for (int kw = 0; kw < 7; ++kw)
#pragma unroll
          for (int q = 0; q < kDwPX; ++q) fma_pair(acc[1][q], v[q + kw], wprev[kw]);
      }
      if (i < 7) {
#pragma unroll
        for (int kw = 0; kw < 7; ++kw) wprev[kw] = wcur[kw];
      }
    }
    uint32_t packed[kDwR][kDwPX];
#pragma unroll
    for (int r = 0; r < kDwR; ++r)
#pragma unroll
      for (int q = 0; q < kDwPX; ++q)
        packed[r][q] = pack_bf16(__uint_as_float(static_cast<uint32_t>(acc[r][q] & 0xffffffffull)), __uint_as_float(static_cast<uint32_t>(acc[r][q] >> 32)));
#pragma unroll
    for (int r = 0; r < kDwR; ++r) {
      const int oh = oh0 + kDwR * rp + r;
      if (oh < p.H && c_ok) {
        uint32_t* yr = reinterpret_cast<uint32_t*>(p.y + (static_cast<long>(b) * p.H + oh) * p.W * p.C + c);
#pragma unroll
        for (int q = 0; q < kDwPX; ++q) {
          const int ow = ow0 + hx * kDwPX + q;
          if (ow < p.W) yr[static_cast<long>(ow) * C2] = packed[r][q];  // a warp writes the 128 contiguous bytes of one pixel's chunk
        }
      }
    }
    if (p.ln_stats) {
      // 32 values per lane (2 rows x 8 pixels x {sum, sumsq} of its channel pair) summed over the 32 lanes with a halving butterfly
      // (31 shuffles instead of 160): lane L ends up with the total of value L = stat * 16 + row * 8 + pixel.
      float a[32];
#pragma unroll
      for (int r = 0; r < kDwR; ++r)
#pragma unroll
        for (int q = 0; q < kDwPX; ++q) {
          const float r0 = bf16lo(packed[r][q]), r1 = bf16hi(packed[r][q]);
          a[r * 8 + q] = r0 + r1;
          a[16 + r * 8 + q] = fmaf(r0, r0, r1 * r1);
        }
#pragma unroll
      for (int half = 16; half >= 1; half >>= 1) {
        const bool up = lane & half;
#pragma unroll
        for (int i = 0; i < half; ++i) {
          const float recv = __shfl_xor_sync(0xffffffffu, up ? a[i] : a[i + half], half);
          a[i] = (up ? a[i + half] : a[i]) + recv;
        }
      }
      const int q = lane & 7, r = (lane >> 3) & 1, stat = lane >> 4;
      const int oh = oh0 + kDwR * rp + r, ow = ow0 + hx * kDwPX + q;
      if (oh < p.H && ow < p.W) {
        unsigned long long* dst = p.ln_stats + ((static_cast<long>(b) * p.H + oh) * p.W + ow) * 2 + stat;
        atomicAdd(dst, static_cast<unsigned long long>(__float2ll_rn(a[0] * kGnFixedScale)));
      }
    }
    __syncthreads();  // every thread has read this stage: thread 0 may refill it (two iterations from now it is waited on again)
  }
}

}  // namespace uc

using namespace uc;

extern "C" int uc_dwconv7(const void* x_bf16, const float* w49, const float* bias, void* y_bf16, int B, int H, int W, int C,
                          void* ln_stats, int* work_counter, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!x_bf16 || !w49 || !bias || !y_bf16) return set_error(UC_EINVAL, "uc_dwconv7: null pointer");
  if (x_bf16 == y_bf16) return set_error(UC_EINVAL, "uc_dwconv7: not an in-place operation");
  if (B < 1 || H < 1 || W < 1 || C < 8 || C % 8) return set_error(UC_EINVAL, "uc_dwconv7: C must be a multiple of 8");
  if (((reinterpret_cast<uintptr_t>(x_bf16) | reinterpret_cast<uintptr_t>(y_bf16) | reinterpret_cast<uintptr_t>(w49)) & 15) ||
      (reinterpret_cast<uintptr_t>(bias) & 7))
    return set_error(UC_EINVAL, "uc_dwconv7: 16-byte aligned maps and taps, 8-byte aligned bias");
  int rc = ensure_driver();
  if (rc) return rc;
  DwParams p;
  memset(&p, 0, sizeof(p));
  {
    uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(W), static_cast<uint64_t>(H), static_cast<uint64_t>(B)};
    uint64_t strides[3] = {static_cast<uint64_t>(C) * 2, static_cast<uint64_t>(W) * C * 2, static_cast<uint64_t>(H) * W * C * 2};
    uint32_t box[4] = {kDwCCH, kDwHW, kDwHH, 1};
    rc = encode_tmap(&p.tmX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x_bf16, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {static_cast<uint64_t>(C), 49};
    uint64_t strides[1] = {static_cast<uint64_t>(C) * 4};
    uint32_t box[2] = {kDwCCH, 49};
    rc = encode_tmap(&p.tmW, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, w49, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
  }
  p.bias = bias;
  p.y = static_cast<uint16_t*>(y_bf16);
  p.ln_stats = static_cast<unsigned long long*>(ln_stats);
  p.work_counter = work_counter;
  p.H = H; p.W = W; p.C = C; p.B = B;
  p.tiles_w = (W + kDwTW - 1) / kDwTW;
  p.tiles_h = (H + kDwTH - 1) / kDwTH;
  const long items = static_cast<long>(p.tiles_w) * p.tiles_h * B * ((C + kDwCCH - 1) / kDwCCH);
  if (items > 0x7fffffffL) return set_error(UC_EINVAL, "uc_dwconv7: too many tiles");
  p.n_items = static_cast<int>(items);
  static PerDeviceFlag attr_dev;
  bool& attr = attr_dev.get();
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(dwconv7_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDwSmem);
    if (e != cudaSuccess) return set_error(static_cast<int>(e), "uc_dwconv7: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr = true;
  }
  const int grid = static_cast<int>(std::min<long>(items, static_cast<long>(num_sms()) * kDwCtasPerSm));
  cudaError_t e = launch_pdl(dwconv7_tma_kernel, dim3(grid), dim3(kDwThreads), kDwSmem, stream, p);
  if (e != cudaSuccess) return set_error(static_cast<int>(e), "uc_dwconv7 launch: %s", cudaGetErrorString(e));
  return check_launch("uc_dwconv7");
}
