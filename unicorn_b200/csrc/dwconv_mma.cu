// Depthwise 7x7 convolution (pad 3) + bias of the ConvNeXt block (unicorn/models/backbone/convnext.py:43) on TENSOR CORES.
//
// The fp32-FMA kernel (dwconv_tma.cu) is bound by FMA issue at ~45 % of a 73 TFLOP/s ceiling (98 flop per output element, 15.6 GFLOP
// per frame).  A depthwise filter has no channel reduction to feed a GEMM with, but each of its 7 filter ROWS is a 1-D correlation
// along W, and a 1-D correlation of 8 outputs with 7 taps is a 16 x 8 banded (Toeplitz) matrix product:
//
//     out[h, w0+n] += sum_k  X[h + kh - 3, w0 - 4 + k] * T_kh[k][n],      T_kh[k][n] = f[kh][k - n - 1]  (0 <= k-n-1 <= 6, else 0)
//
// i.e. one mma.sync.m16n8k16 (bf16 in, fp32 accumulate) per (channel, filter row, 16 x 8 output block): M = 16 output rows, K = a
// 16-pixel window of one input row, N = 8 output columns; 7 MMAs per block and channel, 44 % of the issued MACs are useful, which matters
// little next to the tensor-core rate of mma.sync and the 15.6 GFLOP of useful work per 800x1280 frame.  What it needs is
//   * the input tile CHANNEL-PLANAR in shared memory ([channel][row][col], so that ldmatrix delivers A fragments).  The kernel is
//     bound by shared-memory wavefronts (ldmatrix.x4 = 4), so a warp computes BOTH 8-column blocks of a 16-wide tile from three
//     8-column fragment halves (ldmatrix.x4 + .x2 = 6 wavefronts per two MMAs instead of 8: the middle half is shared);
//   * the B fragments.  Lane (g, t) of a warp holds {T[2t][g], T[2t+1][g]} and {T[2t+8][g], T[2t+9][g]} = the tap pairs
//     (e[d], e[d+1]) and (e[d+8], e[d+9]) with d = 2t - g - 1 and e = the filter row padded with zeros.  Only the 8 pairs
//     (e[j-1], e[j]), j = 0..7, are non-zero, and for a given lane exactly one of its two registers can be (d >= -1: the first,
//     d <= -2: the second), so ONE 32-bit shared-memory load of pair table entry j = d+1 or d+9 and two lane-constant selects give
//     both registers.  The pair table (ops.pack_dw_weight_mma) is 32 B per channel and filter row, 7 KB + the 32 biases per
//     32-channel chunk, and is fetched (one bulk copy) only when a CTA moves to another channel chunk.
//
// Work item = 32 channels x 16 x 16 outputs, CTA = 4 warps, 3 CTAs per SM.  TMA brings the (16+6) x (16+8) x 32-channel NHWC box
// (hardware zero fill = padding) into the staging buffer; the 4 warps transpose it into 32 planes (128-bit loads, conflict-free
// 32-bit stores of pixel pairs thanks to the plane permutation below) and the next item's box is requested as soon as the staging
// buffer is free; warp w = channels 8w .. 8w+7 x the 16 x 16 tile: 56 x (ldmatrix.x4 + ldmatrix.x2 + lds + 2 mma.sync), software
// pipelined over two channels; a lane ends up with 8 consecutive channels of eight pixels = eight 16-byte global stores.  Items are
// handed out by an atomic counter like in dwconv_tma.cu; thread 0 decodes them for everybody.
// Rounding: inputs bf16 (as stored), filter taps bf16 (the FMA kernel keeps them fp32), fp32 accumulation, bf16 output.
#include "uc_ptx.cuh"
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include <algorithm>

namespace uc {

constexpr int kMmTW = 16, kMmTH = 16, kMmCH = 32;
constexpr int kMmHW = kMmTW + 8, kMmHH = kMmTH + 6;                  // 24 x 22 staged box (cols w0-4 .. w0+19, rows oh0-3 .. oh0+18)
constexpr int kMmPixBytes = kMmCH * 2;                                // 64 B per staged pixel
constexpr int kMmStageBytes = kMmHH * kMmHW * kMmPixBytes;           // 33792
constexpr int kMmPlaneBytes = kMmHH * kMmHW * 2;                      // 1056 B = 264 words: 4 consecutive planes start 8 banks apart
constexpr int kMmPlanarBytes = kMmCH * kMmPlaneBytes;                 // 33792
constexpr int kMmPairBytes = kMmCH * 7 * 8 * 4;                       // 7168: tap pair table of one chunk ...
constexpr int kMmQBytes = kMmPairBytes + kMmCH * 4;                   // ... + its 32 biases (fp32) = 7296
constexpr int kMmSmem = kMmStageBytes + kMmPlanarBytes + kMmQBytes + 128 + 128;
constexpr int kMmWarps = 4, kMmCtasPerSm = 3;

struct alignas(64) DwMmaParams {
  CUtensorMap tmX;
  const uint8_t* qtab;  // [ceil(C/32)] x {[32][7][8] int32 tap pairs, [32] fp32 bias}
  uint16_t* y;
  int* work_counter;
  int H, W, C, B, tiles_w, tiles_h, n_items;
};

// physical plane of channel c (0..31): the 4 channel quarters of one transposition store land in 4 CONSECUTIVE planes
__device__ __forceinline__ int mm_plane(int c) { return (c & 7) * 4 + (c >> 3); }

__device__ __forceinline__ void bulk_load_1d(void* smem, const void* gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem)), "l"(gmem),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

struct DwFrag {
  uint32_t a[2][6];  // per channel of the pair: the three 8-column halves {rows 0-7, rows 8-15} x {cols 0-7, 8-15, 16-23}
  uint32_t q[2];
};

__global__ void __launch_bounds__(kMmWarps * 32, kMmCtasPerSm) dwconv7_mma_kernel(const __grid_constant__ DwMmaParams p) {
  constexpr int CPW = kMmCH / kMmWarps;  // 8 channels per warp
  extern __shared__ uint8_t dsm_raw[];
  uint8_t* stage = dsm_raw + ((128u - (smem_u32(dsm_raw) & 127u)) & 127u);
  uint8_t* planar = stage + kMmStageBytes;                                           // [32 planes][22][24] bf16
  uint8_t* qs = planar + kMmPlanarBytes;                                             // tap pairs + biases of the current chunk
  uint64_t* bar = reinterpret_cast<uint64_t*>(qs + kMmQBytes);                       // full, q
  volatile int* s_info = reinterpret_cast<volatile int*>(bar + 2);                   // [2][4]: chunk (-1 = no more items), b, oh0, ow0
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tmX);
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();
  const int tiles_img = p.tiles_w * p.tiles_h, tiles_chunk = tiles_img * p.B;
  int static_next = blockIdx.x;
  auto fetch = [&]() {
    if (p.work_counter) return atomicAdd(p.work_counter, 1);
    const int item = static_next;
    static_next += gridDim.x;
    return item;
  };
  auto issue = [&](int slot, int item) {  // thread 0: decode the item for everybody and request its box
    volatile int* info = s_info + slot * 4;
    if (item >= p.n_items) {
      info[0] = -1;
      mbar_arrive(&bar[0]);
      return;
    }
    const int chunk = item / tiles_chunk, tt0 = item - chunk * tiles_chunk;
    const int b = tt0 / tiles_img, tt = tt0 - b * tiles_img;
    const int oh0 = (tt / p.tiles_w) * kMmTH, ow0 = (tt % p.tiles_w) * kMmTW;
    info[0] = chunk; info[1] = b; info[2] = oh0; info[3] = ow0;
    mbar_arrive_expect_tx(&bar[0], kMmStageBytes);
    tma_load_4d(stage, &p.tmX, &bar[0], chunk * kMmCH, ow0 - 4, oh0 - 3, b);
  };
  int pending = 0;
  if (threadIdx.x == 0) {
    issue(0, fetch());
    pending = fetch();
  }
  // ldmatrix row addresses of this lane inside a plane.  x4: {rows 0-7, cols 0-7}, {rows 8-15, cols 0-7}, {rows 0-7, cols 8-15},
  // {rows 8-15, cols 8-15};  x2: {rows 0-7, cols 16-23}, {rows 8-15, cols 16-23} (lanes 0-15 give the addresses)
  const int fc = warp * CPW;  // first channel of the warp in the chunk; its channel c lives in plane mm_plane(fc + c) = mm_plane(fc) + 4 c
  const uint32_t planar_w = smem_u32(planar) + mm_plane(fc) * kMmPlaneBytes;
  const uint32_t lm4 = planar_w + static_cast<uint32_t>((((lane & 7) + ((lane >> 3) & 1) * 8) * kMmHW + (lane >> 4) * 8) * 2);
  const uint32_t lm2 = planar_w + static_cast<uint32_t>(((lane & 15) * kMmHW + 16) * 2);
  // B fragments from the pair table: entry d+1 feeds the first register (d >= -1), entry d+9 the second (d <= -2)
  const int d = 2 * t - g - 1;
  const bool first = d >= -1;
  const uint32_t q_lane = smem_u32(qs) + static_cast<uint32_t>((fc * 7 * 8 + (first ? d + 1 : d + 9)) * 4);
  const float* bias_s = reinterpret_cast<const float*>(qs + kMmPairBytes) + fc;
  // transposition roles: lane = (pixel pair i, channel quarter q); odd i read their two pixels in the other order (no bank conflict
  // between the 128-byte-strided pairs), which only changes the byte-permute selectors
  const int tq = lane & 3, tsw = (lane >> 2) & 1;
  const uint32_t sel_lo = tsw ? 0x1054u : 0x5410u, sel_hi = tsw ? 0x3276u : 0x7632u;
  auto load_frag = [&](int s, DwFrag& f) {  // step s = channel pair s / 7, filter row s % 7
    const int kh = s % 7;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int c = (s / 7) * 2 + j;
      const uint32_t off = static_cast<uint32_t>(c * 4 * kMmPlaneBytes + kh * (kMmHW * 2));
      asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                   : "=r"(f.a[j][0]), "=r"(f.a[j][1]), "=r"(f.a[j][2]), "=r"(f.a[j][3]) : "r"(lm4 + off));
      asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(f.a[j][4]), "=r"(f.a[j][5]) : "r"(lm2 + off));
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(f.q[j]) : "r"(q_lane + static_cast<uint32_t>((c * 7 + kh) * 32)));
    }
  };
  int prev_chunk = -1;
  uint32_t q_phase = 0;
  for (int it = 0;; ++it) {
    mbar_wait(&bar[0], it & 1);
    const int chunk = s_info[(it & 1) * 4 + 0];
    if (chunk < 0) break;
    const int b = s_info[(it & 1) * 4 + 1], oh0 = s_info[(it & 1) * 4 + 2], ow0 = s_info[(it & 1) * 4 + 3];
    const int c0 = chunk * kMmCH + fc;  // first of this warp's CPW channels
    const bool new_chunk = chunk != prev_chunk;
    prev_chunk = chunk;
    if (new_chunk && threadIdx.x == 0) {  // every warp left the previous item's MMA phase (barrier at the end of the loop body)
      mbar_arrive_expect_tx(&bar[1], kMmQBytes);
      bulk_load_1d(qs, p.qtab + static_cast<size_t>(chunk) * kMmQBytes, kMmQBytes, &bar[1]);
    }
    // ---- NHWC box -> channel planes.  One iteration = 8 pixel pairs x 32 channels per warp: a lane loads 8 channels of two adjacent
    // pixels (2 x 128 bits) and stores 8 words {pixel, pixel + 1} to 8 planes; for a given store the 4 lanes of a pair (the 4 channel
    // quarters) hit 4 consecutive planes = bank groups 0, 8, 16, 24 and the 8 pairs are adjacent words of a plane: conflict free.
    {
      const uint4* st = reinterpret_cast<const uint4*>(stage);
#pragma unroll 3
      for (int pp = warp * 8 + (lane >> 2); pp < kMmHH * kMmHW / 2; pp += kMmWarps * 8) {
        const uint4 va = st[(2 * pp + tsw) * 4 + tq];
        const uint4 vb = st[(2 * pp + (tsw ^ 1)) * 4 + tq];
        const uint32_t wa[4] = {va.x, va.y, va.z, va.w}, wb[4] = {vb.x, vb.y, vb.z, vb.w};
        uint8_t* dst = planar + pp * 4;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint32_t*>(dst + mm_plane(tq * 8 + j) * kMmPlaneBytes) = __byte_perm(wa[j >> 1], wb[j >> 1], j & 1 ? sel_hi : sel_lo);
      }
    }
    __syncthreads();  // planes complete, staging buffer free
    if (threadIdx.x == 0) {
      issue((it + 1) & 1, pending);
      pending = fetch();
    }
    if (new_chunk) {
      mbar_wait(&bar[1], q_phase);
      q_phase ^= 1;
    }
    if (c0 < p.C) {  // C % 8 == 0: the warp's channels are in range together
      // ---- 4 channel pairs x 7 filter rows; per step and channel: 3 fragment halves, 1 tap pair, 2 MMAs (column blocks 0 and 1)
      float acc[CPW][2][4];
#pragma unroll
      for (int c = 0; c < CPW; ++c) {
        const float bv = bias_s[c];
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[c][0][e] = acc[c][1][e] = bv;
      }
      DwFrag fr[2];
      load_frag(0, fr[0]);
#pragma unroll
      for (int s = 0; s < CPW / 2 * 7; ++s) {
        if (s + 1 < CPW / 2 * 7) load_frag(s + 1, fr[(s + 1) & 1]);
        const DwFrag& f = fr[s & 1];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int c = (s / 7) * 2 + j;
          const uint32_t b0 = first ? f.q[j] : 0u, b1 = first ? 0u : f.q[j];
#pragma unroll
          for (int nb = 0; nb < 2; ++nb)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(acc[c][nb][0]), "+f"(acc[c][nb][1]), "+f"(acc[c][nb][2]), "+f"(acc[c][nb][3])
                         : "r"(f.a[j][2 * nb]), "r"(f.a[j][2 * nb + 1]), "r"(f.a[j][2 * nb + 2]), "r"(f.a[j][2 * nb + 3]), "r"(b0), "r"(b1));
        }
      }
      // ---- a lane holds CPW consecutive channels of the pixels (g | g+8, 8 nb + 2t | 2t+1): 16- / 8-byte stores
      uint16_t* yb = p.y + ((static_cast<size_t>(b) * p.H + oh0) * p.W + ow0) * p.C + c0;
#pragma unroll
      for (int nb = 0; nb < 2; ++nb)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int r = g + (e >> 1) * 8, cl = nb * 8 + 2 * t + (e & 1);
          if (oh0 + r < p.H && ow0 + cl < p.W) {
            uint4 o;
            o.x = pack_bf16(acc[0][nb][e], acc[1][nb][e]); o.y = pack_bf16(acc[2][nb][e], acc[3][nb][e]);
            o.z = pack_bf16(acc[4][nb][e], acc[5][nb][e]); o.w = pack_bf16(acc[6][nb][e], acc[7][nb][e]);
            *reinterpret_cast<uint4*>(yb + (static_cast<size_t>(r) * p.W + cl) * p.C) = o;
          }
        }
    }
    __syncthreads();  // the planes and the pair table may be rewritten for the next item
  }
}

}  // namespace uc

using namespace uc;

extern "C" int uc_dwconv7_mma(const void* x_bf16, const void* qtab, void* y_bf16, int B, int H, int W, int C,
                              int* work_counter, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!x_bf16 || !qtab || !y_bf16) return set_error(UC_EINVAL, "uc_dwconv7_mma: null pointer");
  if (x_bf16 == y_bf16) return set_error(UC_EINVAL, "uc_dwconv7_mma: not an in-place operation");
  if (B < 1 || H < 1 || W < 1 || C < 8 || C % 8) return set_error(UC_EINVAL, "uc_dwconv7_mma: C must be a multiple of 8");
  if ((reinterpret_cast<uintptr_t>(x_bf16) | reinterpret_cast<uintptr_t>(y_bf16) | reinterpret_cast<uintptr_t>(qtab)) & 15) return set_error(UC_EINVAL, "uc_dwconv7_mma: 16-byte aligned maps");
  int rc = ensure_driver();
  if (rc) return rc;
  DwMmaParams p;
  memset(&p, 0, sizeof(p));
  {
    uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(W), static_cast<uint64_t>(H), static_cast<uint64_t>(B)};
    uint64_t strides[3] = {static_cast<uint64_t>(C) * 2, static_cast<uint64_t>(W) * C * 2, static_cast<uint64_t>(H) * W * C * 2};
    uint32_t box[4] = {kMmCH, kMmHW, kMmHH, 1};
    rc = encode_tmap(&p.tmX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, x_bf16, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
    if (rc) return rc;
  }
  p.qtab = static_cast<const uint8_t*>(qtab);
  p.y = static_cast<uint16_t*>(y_bf16);
  p.work_counter = work_counter;
  p.H = H; p.W = W; p.C = C; p.B = B;
  p.tiles_w = (W + kMmTW - 1) / kMmTW;
  p.tiles_h = (H + kMmTH - 1) / kMmTH;
  const long items = static_cast<long>(p.tiles_w) * p.tiles_h * B * ((C + kMmCH - 1) / kMmCH);
  if (items > 0x7fffffffL) return set_error(UC_EINVAL, "uc_dwconv7_mma: too many tiles");
  p.n_items = static_cast<int>(items);
  static PerDeviceFlag attr_dev;
  bool& attr = attr_dev.get();
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(dwconv7_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMmSmem);
    if (e != cudaSuccess) return set_error(static_cast<int>(e), "uc_dwconv7_mma: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr = true;
  }
  const int grid = static_cast<int>(std::min<long>(items, static_cast<long>(num_sms()) * kMmCtasPerSm));
  cudaError_t e = launch_pdl(dwconv7_mma_kernel, dim3(grid), dim3(kMmWarps * 32), kMmSmem, stream, p);
  if (e != cudaSuccess) return set_error(static_cast<int>(e), "uc_dwconv7_mma launch: %s", cudaGetErrorString(e));
  return check_launch("uc_dwconv7_mma");
}
