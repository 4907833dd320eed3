// Fused ConvNeXt block back half (unicorn/models/backbone/convnext.py:45-52):
//
//     x += gamma * ( W2 . GELU( W1 . LayerNorm(t) + b1 ) + b2 )          t = depthwise-conv output, x = the block's input (shortcut)
//
// in ONE persistent launch for C = 96, 192, 256, 384 (stages 1-2 of ConvNeXt-L, stages 1-3 of ConvNeXt-T, the attention blocks of
// the head).  There the separate
// kernels are bound by the 4C hidden map, which pwconv1 writes to and pwconv2 reads back from HBM, and by the LayerNorm pass; here
// the hidden activations never leave the SM:
//
//   * TMA brings a 128-row x C tile of t into 128B-swizzled shared memory (K-major wgmma operand layout); each consumer warpgroup
//     LayerNorms its 64 rows IN PLACE (two-pass mean / variance in fp32 over the bf16 values, like uc_layernorm; the affine part is
//     folded into W1 / b1 by the host: W1' = W1 diag(g), b1' = b1 + W1 beta) and publishes them to the tensor core with a proxy fence;
//   * the hidden dimension is walked in chunks of 64: GEMM1 (wgmma 64 x 64 x 16, K = C, both operands in shared memory) -> registers
//     -> + b1', exact GELU (uc_epilogue.cuh), rounded to bf16 IN REGISTERS: the fp32 accumulator fragment of GEMM1 is, pair by pair,
//     the A-operand fragment of GEMM2 (wgmma 64 x C x 16 with A from registers, K = 64), which accumulates into the output registers;
//     the weight chunks W1'[64 j .. 64 j + 63][:] and W2[:][64 j .. 64 j + 63] stream through two TMA rings;
//   * C = 384: the 64 x 384 output accumulator does not fit a warpgroup's registers next to the hidden chunk, so the output columns
//     are computed in two halves of 192, each walking all hidden chunks (GEMM1 and the GELU are evaluated twice);
//   * after the last chunk the warpgroup adds b2 to its accumulator, multiplies by the layer scale, adds the shortcut and stores x
//     in place — the same epilogue arithmetic and order as uc_conv2d's.  Every shortcut load of the tile is issued right before the
//     last chunk's GEMM2 and ahead of the first store, so the loads run under that GEMM2: a load behind a store to the same map
//     would wait for it, one memory round trip per 8-column group and row half.  b2 and the layer scale are read from a copy in
//     shared memory.
//   * the two consumer warpgroups share the weight rings and run independently otherwise, so one is in its GELU / LayerNorm while
//     the other keeps the tensor core busy.
//
// Warp roles (384 threads, 1 CTA / SM): warpgroup 0 = TMA producer (one warp), warpgroups 1-2 = rows 0-63 / 64-127 of the tile.
#include <algorithm>
#include "uc_ptx.cuh"
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include "uc_epilogue.cuh"

namespace uc {

constexpr int kMlpRows = 128;
constexpr int kMlpHC = 64;  // hidden chunk = one 128-byte K block of GEMM2
constexpr int kMlpConsumers = 2;
constexpr int kMlpThreads = (1 + kMlpConsumers) * 128;

template <int C>
struct MlpCfg {
  static constexpr int KB = (C + 63) / 64;              // K blocks of the row tile (the last one zero-filled past C by TMA)
  static constexpr int A_BYTES = KB * kMlpRows * 128;   // 128 rows x KB x 128 B
  static constexpr int W1_BYTES = KB * kMlpHC * 128;    // 64 hidden rows x KB x 128 B
  static constexpr int NH = C > 256 ? 2 : 1;            // output column halves (register budget, see above)
  static constexpr int N2 = C / NH;                     // output columns per pass
  static constexpr int W2_BYTES = N2 * 128;             // N2 output rows x 64 hidden (128 B)
  static constexpr int NCHUNK = 4 * C / kMlpHC;
  static constexpr int STEPS = NH * NCHUNK;             // weight chunks per row tile
  static constexpr int AS = C <= 192 ? 2 : 1;           // row-tile buffers (C >= 256 has room for one next to the weight rings)
  static constexpr int WS = C <= 256 ? 2 : 1;           // weight-ring stages
  static constexpr int SMEM = AS * A_BYTES + WS * (W1_BYTES + W2_BYTES) + 1024 + 512 + 2 * C * 4;  // + barriers, b2 / gamma
  static constexpr int CPT = C / 16;                    // 16-byte chunks of a row per LayerNorm thread (2 threads per row)
};

struct alignas(64) MlpParams {
  CUtensorMap tmA, tmW1, tmW2;
  const float* c1;     // [4C] folded bias of pwconv1
  const float* b2;     // [C]
  const float* gamma;  // [C] layer scale
  uint16_t* x;         // [M][C] shortcut in, block output out
  int M, m_tiles;
  float ln_eps;
};

// barrier indices
enum { A_FULL = 0, A_EMPTY = 2, W1_FULL = 4, W1_EMPTY = 6, W2_FULL = 8, W2_EMPTY = 10, MLP_NBARS = 12 };

template <int C>
__global__ void __launch_bounds__(kMlpThreads, 1) convnext_mlp_kernel(const __grid_constant__ MlpParams p) {
  using Cfg = MlpCfg<C>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                                 // [AS][KB][128 rows][128 B]
  uint8_t* sW1 = sA + Cfg::AS * Cfg::A_BYTES;         // [WS][KB][64 rows][128 B]
  uint8_t* sW2 = sW1 + Cfg::WS * Cfg::W1_BYTES;       // [WS][C rows][128 B]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sW2 + Cfg::WS * Cfg::W2_BYTES);
  // [C] b2, then [C] gamma; addressed from smem_raw so that the compiler reads them with LDS
  float* sB2 = reinterpret_cast<float*>(smem_raw + (sW2 + Cfg::WS * Cfg::W2_BYTES + 512 - smem_raw));
  float* sGm = sB2 + C;
  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tmA);
    prefetch_tmap(&p.tmW1);
    prefetch_tmap(&p.tmW2);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&bar[A_FULL + i], 1);
      mbar_init(&bar[A_EMPTY + i], kMlpConsumers);
      mbar_init(&bar[W1_FULL + i], 1);
      mbar_init(&bar[W1_EMPTY + i], kMlpConsumers);
      mbar_init(&bar[W2_FULL + i], 1);
      mbar_init(&bar[W2_EMPTY + i], kMlpConsumers);
    }
    fence_barrier_init();
  }
  pdl_wait();
  pdl_launch_dependents();
  static_assert(C <= kMlpThreads, "one b2 / gamma column per thread");
  if (threadIdx.x < C) {
    sB2[threadIdx.x] = p.b2[threadIdx.x];
    sGm[threadIdx.x] = p.gamma[threadIdx.x];
  }
  __syncthreads();

  const int n_local = (p.m_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);  // row tiles of this CTA
  auto tile_of = [&](int i) { return static_cast<int>(blockIdx.x) + i * static_cast<int>(gridDim.x); };

  if (wg == 0) {
    regs_dealloc<40>();
    if (warp != 0) return;
    // ---------------- TMA producer
    auto load_a = [&](int i) {
      const int ab = i % Cfg::AS;
      mbar_wait(&bar[A_EMPTY + ab], ((i / Cfg::AS) & 1) ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&bar[A_FULL + ab], Cfg::A_BYTES);
#pragma unroll
        for (int kb = 0; kb < Cfg::KB; ++kb)
          tma_load_2d(sA + ab * Cfg::A_BYTES + kb * (kMlpRows * 128), &p.tmA, &bar[A_FULL + ab], kb * 64, tile_of(i) * kMlpRows);
      }
      __syncwarp();
    };
    // weight step g: hidden rows (W1) / columns (W2) 64 j .. + 63 of output half nh
    auto load_w = [&](int g) {
      const int s = g % Cfg::WS, ph = (g / Cfg::WS) & 1, j = g % Cfg::NCHUNK, nh = (g / Cfg::NCHUNK) % Cfg::NH;
      mbar_wait(&bar[W1_EMPTY + s], ph ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&bar[W1_FULL + s], Cfg::W1_BYTES);
#pragma unroll
        for (int kb = 0; kb < Cfg::KB; ++kb)
          tma_load_2d(sW1 + s * Cfg::W1_BYTES + kb * (kMlpHC * 128), &p.tmW1, &bar[W1_FULL + s], kb * 64, j * kMlpHC);
      }
      __syncwarp();
      mbar_wait(&bar[W2_EMPTY + s], ph ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&bar[W2_FULL + s], Cfg::W2_BYTES);
        tma_load_2d(sW2 + s * Cfg::W2_BYTES, &p.tmW2, &bar[W2_FULL + s], j * kMlpHC, nh * Cfg::N2);
      }
      __syncwarp();
    };
    const int total = n_local * Cfg::STEPS;
    if (n_local > 0) load_a(0);
    for (int g = 0; g < total; ++g) {
      load_w(g);
      const int i = g / Cfg::STEPS, r = g % Cfg::STEPS;
      // the next row tile: into the other buffer right away, or (single buffer) once the last GEMM1 of this tile has read it
      if (r == (Cfg::AS == 2 ? 0 : Cfg::STEPS - 1) && i + 1 < n_local) load_a(i + 1);
    }
    return;
  }
  regs_alloc<232>();
  // ---------------- consumer warpgroup c: rows 64c .. 64c+63 of every row tile.  Accumulator fragment of thread (warp w of the
  // warpgroup, lane = 4 g + t): rows 16 w + g and 16 w + g + 8, columns 8i + 2t, 8i + 2t + 1 in registers 4i .. 4i+3.
  const int c = wg - 1, ct = threadIdx.x & 127;
  const int g8 = lane >> 2, t = lane & 3;
  const int rl = (warp & 3) * 16 + g8;  // first row of this thread inside the warpgroup's 64
  // LayerNorm: 2 threads per row (adjacent lanes), part lp handles the 16-byte chunks lp * CPT .. + CPT - 1
  const int lr = c * 64 + (ct >> 1), lp = ct & 1;
  auto layer_norm_tile = [&](int ab) {
    uint8_t* a = sA + ab * Cfg::A_BYTES + lr * 128;
    // chunk gc of the row: K block gc / 8, 16-byte slot gc % 8 (swizzled with the row)
    auto chunk_ptr = [&](int cc) {
      const int gc = lp * Cfg::CPT + cc;
      return reinterpret_cast<uint4*>(a + (gc >> 3) * (kMlpRows * 128) + (((gc & 7) ^ (lr & 7)) << 4));
    };
    float s1 = 0.f;
#pragma unroll 4
    for (int cc = 0; cc < Cfg::CPT; ++cc) {
      const uint4 v = *chunk_ptr(cc);
      s1 += (bf16lo(v.x) + bf16hi(v.x)) + (bf16lo(v.y) + bf16hi(v.y)) + (bf16lo(v.z) + bf16hi(v.z)) + (bf16lo(v.w) + bf16hi(v.w));
    }
    s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
    const float mean = s1 * (1.f / C);
    float s2 = 0.f;
#pragma unroll 4
    for (int cc = 0; cc < Cfg::CPT; ++cc) {
      const uint4 v = *chunk_ptr(cc);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float d0 = bf16lo(w[e]) - mean, d1 = bf16hi(w[e]) - mean;
        s2 = fmaf(d0, d0, s2);
        s2 = fmaf(d1, d1, s2);
      }
    }
    s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
    const float rstd = rsqrtf(s2 * (1.f / C) + p.ln_eps);
#pragma unroll 4
    for (int cc = 0; cc < Cfg::CPT; ++cc) {
      uint4* ptr = chunk_ptr(cc);
      const uint4 v = *ptr;
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      uint32_t o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) o[e] = pack2_fast((bf16lo(w[e]) - mean) * rstd, (bf16hi(w[e]) - mean) * rstd, false);
      *ptr = make_uint4(o[0], o[1], o[2], o[3]);
    }
    fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
    named_sync(1 + c, 128);
  };
  const uint64_t a_desc0 = wgmma_desc_sw128(smem_u32(sA + c * 64 * 128)), w1_desc0 = wgmma_desc_sw128(smem_u32(sW1));
  const uint64_t w2_desc0 = wgmma_desc_sw128(smem_u32(sW2));
  float acc2[Cfg::N2 / 2];
  uint32_t hf[4][4];  // GEMM2's A fragment: the bf16 hidden chunk
  // ---- GEMM2 of weight step (ws, wph): output accumulator += H chunk . W2 chunk^T
  auto gemm2 = [&](int j, int ws, int wph) {
    mbar_wait(&bar[W2_FULL + ws], wph);
    wgmma_fence();
    const uint64_t bd2 = w2_desc0 + static_cast<uint64_t>((ws * Cfg::W2_BYTES) >> 4);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs_bf16<Cfg::N2>(acc2, hf[kk], bd2 + 2 * kk, (j | kk) != 0 ? 1u : 0u);
    wgmma_commit();
  };
  int g = 0;
  for (int i = 0; i < n_local; ++i) {
    const int ab = i % Cfg::AS;
    mbar_wait(&bar[A_FULL + ab], (i / Cfg::AS) & 1);
    layer_norm_tile(ab);
#pragma unroll 1
   for (int nh = 0; nh < Cfg::NH; ++nh) {
    int ws, wph;
    for (int j = 0;; ++j, ++g) {
      ws = g % Cfg::WS;
      wph = (g / Cfg::WS) & 1;
      // ---- GEMM1: hidden chunk j of this warpgroup's 64 rows
      float acc1[kMlpHC / 2];
      mbar_wait(&bar[W1_FULL + ws], wph);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < Cfg::KB; ++kb) {
        const uint64_t ad = a_desc0 + static_cast<uint64_t>((ab * Cfg::A_BYTES + kb * (kMlpRows * 128)) >> 4);
        const uint64_t bd = w1_desc0 + static_cast<uint64_t>((ws * Cfg::W1_BYTES + kb * (kMlpHC * 128)) >> 4);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<kMlpHC, false>(acc1, ad + 2 * k, bd + 2 * k, (kb | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc1);
      if (ct == 0) {
        mbar_arrive(&bar[W1_EMPTY + ws]);
        if (nh == Cfg::NH - 1 && j == Cfg::NCHUNK - 1) mbar_arrive(&bar[A_EMPTY + ab]);
      }
      // ---- + b1', GELU, bf16: accumulator columns 16 kk .. 16 kk + 15 are the A fragment of GEMM2's K step kk
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int i8 = 2 * kk + half;
          const float2 bb = __ldg(reinterpret_cast<const float2*>(p.c1 + j * kMlpHC + 8 * i8 + 2 * t));
          const f32x2 h0 = gelu2(add2(pk2(acc1[4 * i8], acc1[4 * i8 + 1]), pk2(bb.x, bb.y)));
          const f32x2 h1 = gelu2(add2(pk2(acc1[4 * i8 + 2], acc1[4 * i8 + 3]), pk2(bb.x, bb.y)));
          hf[kk][2 * half] = pack2_fast(lo2(h0), hi2(h0), false);
          hf[kk][2 * half + 1] = pack2_fast(lo2(h1), hi2(h1), false);
        }
      }
      if (j == Cfg::NCHUNK - 1) break;  // the last chunk's GEMM2 is issued below, behind the shortcut loads
      gemm2(j, ws, wph);
      wgmma_wait<0>();
      wgmma_fence_regs(acc2);
      if (ct == 0) mbar_arrive(&bar[W2_EMPTY + ws]);
    }
    // ---- output columns nh * N2 .. : x += gamma * (acc2 + b2).  The shortcut words of both row halves of every 8-column group
    // are loaded first, all of them before the first store (rows past M are neither read nor written), and run under the last
    // chunk's GEMM2.  They are issued ahead of it, not behind it: a register written while an RS wgmma is in flight may be one
    // of hf's, and ptxas then waits for the wgmma before the write.
    const long grow0 = static_cast<long>(tile_of(i)) * kMlpRows + c * 64 + rl;
    uint32_t* xr = reinterpret_cast<uint32_t*>(p.x + grow0 * C + nh * Cfg::N2 + 2 * t);
    const bool in0 = grow0 < p.M, in1 = grow0 + 8 < p.M;
    uint32_t rw[Cfg::N2 / 4];
#pragma unroll
    for (int i8 = 0; i8 < Cfg::N2 / 8; ++i8) {
      rw[2 * i8] = in0 ? xr[4 * i8] : 0u;
      rw[2 * i8 + 1] = in1 ? xr[4 * i8 + 4 * C] : 0u;
    }
    gemm2(Cfg::NCHUNK - 1, ws, wph);
    wgmma_wait<0>();
    wgmma_fence_regs(acc2);
    if (ct == 0) mbar_arrive(&bar[W2_EMPTY + ws]);
    ++g;
#pragma unroll
    for (int i8 = 0; i8 < Cfg::N2 / 8; ++i8) {
      const int col = nh * Cfg::N2 + 8 * i8 + 2 * t;
      const float2 b = *reinterpret_cast<const float2*>(sB2 + col), gm = *reinterpret_cast<const float2*>(sGm + col);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (h == 0 ? in0 : in1) {
          f32x2 v = add2(pk2(acc2[4 * i8 + 2 * h], acc2[4 * i8 + 2 * h + 1]), pk2(b.x, b.y));
          v = mul2(v, pk2(gm.x, gm.y));
          v = add2(v, pk2(bf16lo(rw[2 * i8 + h]), bf16hi(rw[2 * i8 + h])));
          xr[4 * i8 + 4 * C * h] = pack2_fast(lo2(v), hi2(v), false);
        }
      }
    }
   }
  }
}

template <int C>
static int launch_mlp(MlpParams& p, cudaStream_t stream) {
  using Cfg = MlpCfg<C>;
  static PerDeviceFlag attr_dev;
  bool& attr = attr_dev.get();
  auto kern = convnext_mlp_kernel<C>;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return set_error(static_cast<int>(e), "uc_convnext_mlp: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr = true;
  }
  const int grid = std::min(p.m_tiles, num_sms());
  cudaError_t e = launch_pdl(kern, dim3(grid), dim3(kMlpThreads), Cfg::SMEM, stream, p);
  if (e != cudaSuccess) return set_error(static_cast<int>(e), "uc_convnext_mlp<%d> launch: %s", C, cudaGetErrorString(e));
  return check_launch("uc_convnext_mlp");
}

}  // namespace uc

using namespace uc;

extern "C" int uc_convnext_mlp_supported(int C) { return C == 96 || C == 192 || C == 256 || C == 384; }

extern "C" int uc_convnext_mlp(const void* t_bf16, const void* w1f_bf16, const float* c1, const void* w2_bf16, const float* b2,
                               const float* gamma, void* x_bf16, int M, int C, float ln_eps, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!t_bf16 || !w1f_bf16 || !c1 || !w2_bf16 || !b2 || !gamma || !x_bf16) return set_error(UC_EINVAL, "uc_convnext_mlp: null pointer");
  if (!uc_convnext_mlp_supported(C)) return set_error(UC_EINVAL, "uc_convnext_mlp: C = %d not supported (96, 192, 256, 384)", C);
  if (M < 1) return set_error(UC_EINVAL, "uc_convnext_mlp: empty map");
  if ((reinterpret_cast<uintptr_t>(t_bf16) | reinterpret_cast<uintptr_t>(w1f_bf16) | reinterpret_cast<uintptr_t>(w2_bf16)) & 15 ||
      (reinterpret_cast<uintptr_t>(x_bf16) | reinterpret_cast<uintptr_t>(c1) | reinterpret_cast<uintptr_t>(b2) | reinterpret_cast<uintptr_t>(gamma)) & 31)
    return set_error(UC_EINVAL, "uc_convnext_mlp: t / weights 16-byte, x / biases 32-byte aligned");
  if (t_bf16 == x_bf16) return set_error(UC_EINVAL, "uc_convnext_mlp: t and x must be different maps");
  int rc = ensure_driver();
  if (rc) return rc;
  MlpParams p;
  memset(&p, 0, sizeof(p));
  const uint64_t es = 2;
  {
    uint64_t dims[2] = {static_cast<uint64_t>(C), static_cast<uint64_t>(M)};
    uint64_t strides[1] = {static_cast<uint64_t>(C) * es};
    uint32_t box[2] = {64, kMlpRows};
    rc = encode_tmap(&p.tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, t_bf16, dims, strides, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {static_cast<uint64_t>(C), static_cast<uint64_t>(4 * C)};
    uint64_t strides[1] = {static_cast<uint64_t>(C) * es};
    uint32_t box[2] = {64, kMlpHC};
    rc = encode_tmap(&p.tmW1, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, w1f_bf16, dims, strides, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {static_cast<uint64_t>(4 * C), static_cast<uint64_t>(C)};
    uint64_t strides[1] = {static_cast<uint64_t>(4 * C) * es};
    uint32_t box[2] = {kMlpHC, static_cast<uint32_t>(C > 256 ? C / 2 : C)};
    rc = encode_tmap(&p.tmW2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, w2_bf16, dims, strides, box);
    if (rc) return rc;
  }
  p.c1 = c1; p.b2 = b2; p.gamma = gamma;
  p.x = static_cast<uint16_t*>(x_bf16);
  p.M = M;
  p.m_tiles = (M + kMlpRows - 1) / kMlpRows;
  p.ln_eps = ln_eps;
  return C == 96 ? launch_mlp<96>(p, stream) : C == 192 ? launch_mlp<192>(p, stream) : C == 256 ? launch_mlp<256>(p, stream) : launch_mlp<384>(p, stream);
}
