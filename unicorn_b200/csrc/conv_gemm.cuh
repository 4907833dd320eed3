// Implicit-GEMM convolution / linear layer on Hopper tensor cores (wgmma).
//
//   D[pixel, cout] = sum_{tap, cin} X[pixel + tap, cin] * W[cout, tap, cin]
//
// One CTA computes a 128-pixel x BLOCK_N-channel output tile.  The 128 pixels are a tile_w x tile_h patch of
// the NHWC output map; for every filter tap the TMA engine fetches the shifted tile_w x tile_h x 64-channel
// box of the input straight into 128B-swizzled shared memory (out-of-bounds coordinates are zero-filled by
// the hardware, which is the convolution's zero padding), so no im2col buffer ever exists.  Two consumer
// warpgroups own 64 pixels each and issue wgmma m64 x BLOCK_N x 16 (bf16/fp16 in, fp32 accumulate in registers)
// on the shared stage; when a tile's K loop is done they apply bias / activation / layer-scale+residual, and
// optionally accumulate GroupNorm statistics, straight from the accumulator registers, while the producer is
// already filling the ring with the next tile's boxes.
//
// 16-bit outputs leave through a shared-memory staging tile (128 rows x BLOCK_N, slabs of SLAB columns in the swizzled layout
// of a TMA box {SLAB, tile_w, tile_h, 1}).  An epilogue DMA warp loads the tile's residual into it by TMA, and the tile's bias,
// layer-scale and folded-LayerNorm column slices into small shared arrays, while the consumers still run the K loop; so the
// epilogue waits on nothing global.  The consumers overwrite the residual with the output in place and the DMA warp stores the
// tile by TMA (out-of-range rows and columns >= Cout are clipped by the hardware).  An in-place residual (res == y) is safe:
// a tile's residual is read before that tile's store is issued, and tiles are disjoint.  fp32 outputs are stored directly.
//
// CLUSTER = 2 (block_n 1128 / 1192 / 1256): two CTAs of a thread-block cluster take consecutive M tiles of the same N tile.
// Each loads its own activation box and HALF of the weight box, multicast by TMA into the same stage of both CTAs, so the
// weights of a tile are read from L2 once per pair; a stage is refilled when the consumers of BOTH CTAs have released it
// (remote mbarrier arrives).
//
// The epilogue's features are a template parameter (ConvEpi): the unrolled epilogue loop of an instantiation holds only what that
// variant does.  Runtime feature tests inside the loop are repeated BLOCK_N / 8 times, and a kernel carrying all of them is several
// times the size of a single variant's (DESIGN §4.1).  The instantiations are split over several conv_gemm_*.cu files, which compile
// in parallel; conv_gemm.cu holds the host side and picks the instantiation.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (warp 0) and epilogue DMA (warp 1), warpgroups 1-2 = MMA + epilogue.
// Reference call sites replaced: see include/unicorn_b200.h (uc_conv2d).
#pragma once
#include <algorithm>
#include <stdlib.h>
#include "uc_ptx.cuh"
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include "uc_epilogue.cuh"

namespace uc {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 16-bit elements -> 128-byte rows
constexpr int kMaxTaps = 9;
constexpr int kABytes = kBlockM * kBlockK * 2;
constexpr int kConvConsumers = 2;                       // warpgroups of 64 pixels
constexpr int kConvThreads = (1 + kConvConsumers) * 128;
constexpr int kGnMaxLocal = 64;                         // GroupNorm groups per N tile (tile width 256 / group size >= 4)
constexpr int kGnSmemBytes = 2 * kGnMaxLocal * 2 * 8;   // two tile parities x {sum, sumsq} int64
constexpr int kEpiBar = 2;                              // named barrier: consumers have staged a tile (id 1 is the GroupNorm one)

// columns per staging slab: a 128-byte (64), 64-byte (32) or 32-byte (16) swizzled TMA box row that tiles BLOCK_N exactly
constexpr int conv_slab(int block_n) { return block_n % 64 == 0 ? 64 : block_n % 32 == 0 ? 32 : 16; }
// stage ring, 16-bit output staging tile, alignment slack, barriers, GroupNorm slots, bias / gamma / col_s slices, GroupNorm
// local group index per column
constexpr int conv_smem_bytes(int block_n, int stages) {
  return stages * (kABytes + block_n * kBlockK * 2) + kBlockM * block_n * 2 + 1024 + 256 + kGnSmemBytes + 3 * block_n * 4 + block_n;
}

// Epilogue variants.  Each fixed variant is branch-free in the unrolled loop and exists for bf16 operands only; kEpiAny tests every
// feature at run time and takes whatever the others do not cover (f16 operands, SiLU / sigmoid, gamma without a residual, ...).
enum ConvEpi : int {
  kEpiAny = 0,
  kEpiBias,     // + bias, bf16 out (the downsample convs)
  kEpiBiasF16,  // + bias, f16 out (embedding up3)
  kEpiF32,      // + bias, fp32 out (the prediction convs)
  kEpiRelu,     // relu(. + bias), bf16 out
  kEpiGelu,     // gelu(. + bias), bf16 out (pwconv1)
  kEpiGeluLn,   // gelu(folded LayerNorm + bias), bf16 out (pwconv1 with row_stats)
  kEpiRes,      // res + gamma * (. + bias), bf16 out (pwconv2; gamma 1.0 when absent)
  kEpiReluRes,  // relu(. + bias + res), bf16 out (ResNet Bottleneck conv3)
  kEpiGn,       // + bias and GroupNorm statistics, bf16 out (conv_gn)
};

struct ConvTap {
  int16_t map, dw, dh, tap;
};

struct alignas(64) ConvKernelParams {
  CUtensorMap tmA[4];
  CUtensorMap tmB;
  CUtensorMap tmBh;  // half-height weight box of the cluster variant
  CUtensorMap tmY, tmR;  // 16-bit output and residual {Cout, Wo, Ho, B}, box {SLAB, tile_w, tile_h, 1}
  ConvTap taps[kMaxTaps];
  int ntaps, kchunks;
  int n_tiles, m_tiles;
  int tile_w, tile_h, tiles_w, tiles_h;
  int Wo, Ho, B, Cout;
  const float* bias;
  const float* gamma;
  const void* res;
  int ldres;
  void* y;
  int ldy, y_dtype, act;
  int relu_res;  // y = relu(acc + bias + res) (ResNet Bottleneck; act is NONE then)
  const long long* row_stats;  // LayerNorm folded into this 1x1 conv: per input pixel {sum, sumsq} (fixed point 2^22) ...
  const float* col_s;          // ... column sums of the folded weights, channel count and epsilon of the LayerNorm
  float row_inv, row_eps;  // row_inv = 1 / (2^22 * Cin)
  long long* gn_stats;  // fixed-point (2^22) accumulators: order-independent, hence deterministic
  int gn_groups, gn_gs;  // gs = Cout / groups
};

// 64-bit add to shared memory as two native 32-bit atomics.  sm_90 has no 64-bit shared-memory atomic add: atomicAdd on a 64-bit
// shared word compiles to a compare-and-swap loop, which serializes the lanes of all warps that add to one GroupNorm slot.  The lane
// whose add wraps the low word adds the carry to the high word, so once every adder is done (the barrier before the slot is read)
// the slot holds the exact sum modulo 2^64, the same bits as 64-bit atomics in any order.
__device__ __forceinline__ void smem_add_u64(unsigned long long* slot, unsigned long long v) {
  unsigned int* w = reinterpret_cast<unsigned int*>(slot);
  const unsigned int lo = static_cast<unsigned int>(v);
  const unsigned int old = atomicAdd(w, lo);
  atomicAdd(w + 1, static_cast<unsigned int>(v >> 32) + (old + lo < old ? 1u : 0u));
}

// Persistent kernel: grid = min(#tiles, SMs); every CTA (pair) walks work items item = blockIdx.x / CLUSTER + i * gridDim.x / CLUSTER
// (N tile fastest, so CTAs running side by side share the activation tile in L2); item = (N tile, group of CLUSTER M tiles).
template <int BLOCK_N, int STAGES, bool F16, int CLUSTER, int EPI>
__global__ void __launch_bounds__(kConvThreads, 1) conv_gemm_kernel(const __grid_constant__ ConvKernelParams p) {
  constexpr int B_BYTES = BLOCK_N * kBlockK * 2;
  constexpr int NACC = BLOCK_N / 2;  // accumulator registers per thread: m64 x BLOCK_N over 128 threads
  constexpr int SLAB = conv_slab(BLOCK_N), SLAB_BYTES = kBlockM * SLAB * 2;
  constexpr bool ANY = EPI == kEpiAny;
  extern __shared__ uint8_t smem_raw[];
  // offset from the shared window address, not a round trip through an integer: the compiler then knows every pointer below is
  // shared and emits LDS / STS / ATOMS rather than generic accesses
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = sA + STAGES * kABytes;
  uint8_t* sY = sB + STAGES * B_BYTES;  // 16-bit output staging tile (1024-byte aligned, as the 128-byte swizzle needs)
  uint64_t* full = reinterpret_cast<uint64_t*>(sY + kBlockM * BLOCK_N * 2);
  uint64_t* empty = full + STAGES;
  uint64_t* epi_full = empty + STAGES;  // the tile's residual and column slices are in shared memory
  // per-CTA GroupNorm accumulators (fixed point): the epilogue adds into shared memory, ONE global atomic per group and tile
  // follows (the short-K GN convs are otherwise bound by global atomics on the few addresses of an image)
  unsigned long long* gn_acc = reinterpret_cast<unsigned long long*>(reinterpret_cast<uint8_t*>(full) + 256);
  float* s_bias = reinterpret_cast<float*>(gn_acc + 2 * kGnMaxLocal * 2);
  float* s_gamma = s_bias + BLOCK_N;
  float* s_cols = s_gamma + BLOCK_N;
  uint8_t* s_grp = reinterpret_cast<uint8_t*>(s_cols + BLOCK_N);  // GroupNorm group of each tile column, relative to the tile's first

  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kiters = p.ntaps * p.kchunks;
  const int crank = CLUSTER > 1 ? static_cast<int>(cluster_ctarank()) : 0;
  const int num_items = p.n_tiles * ((p.m_tiles + CLUSTER - 1) / CLUSTER);
  const int item0 = blockIdx.x / CLUSTER, item_step = gridDim.x / CLUSTER;
  // the epilogue's features: compile-time constants except in kEpiAny
  const bool use_ln = EPI == kEpiGeluLn || (ANY && p.row_stats);
  const bool use_gn = EPI == kEpiGn || (ANY && p.gn_stats);
  // releases stage s: in the cluster variant the peer's producer multicasts into this CTA's stage too, so both CTAs' rings hear it
  auto release = [&](int s) {
    mbar_arrive(&empty[s]);
    if (CLUSTER > 1) mbar_arrive_remote(&empty[s], static_cast<uint32_t>(crank ^ 1));
  };

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tmA[0]);
    prefetch_tmap(&p.tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], kConvConsumers * CLUSTER);
    }
    mbar_init(epi_full, 32);  // every lane of the DMA warp (their column-slice writes are released by their own arrive)
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 2 * kGnMaxLocal * 2; i += kConvThreads) gn_acc[i] = 0ull;
  // N tiles start on a group boundary (BLOCK_N % gs == 0), so the local group of a column is the same in every tile
  if (use_gn && threadIdx.x < BLOCK_N) s_grp[threadIdx.x] = static_cast<uint8_t>(threadIdx.x / p.gn_gs);
  __syncthreads();
  if (CLUSTER > 1) cluster_sync_all();  // the peer's barriers are initialised before anything is multicast / arrived to them
  // Programmatic dependent launch: the set-up above overlapped the tail of the previous kernel in the stream; global memory
  // is touched only after it has completed.
  pdl_wait();
  pdl_launch_dependents();

  if (wg == 0) {
    regs_dealloc<40>();
  }
  if (warp == 0) {
    // ---------------- TMA producer: the whole warp walks the loop (converged), one elected lane issues
    int stage = 0, phase = 0;
    for (int item = item0; item < num_items; item += item_step) {
      const int n0 = (item % p.n_tiles) * BLOCK_N;
      const int mt = (item / p.n_tiles) * CLUSTER + crank;
      const int ow0 = (mt % p.tiles_w) * p.tile_w, oh0 = ((mt / p.tiles_w) % p.tiles_h) * p.tile_h;
      const int b = mt / (p.tiles_w * p.tiles_h);
      for (int t = 0; t < p.ntaps; ++t) {
        const ConvTap tp = p.taps[t];
        for (int kc = 0; kc < p.kchunks; ++kc) {
          mbar_wait(&empty[stage], phase ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(&full[stage], kABytes + B_BYTES);  // cluster variant: own A + both multicast weight halves
            tma_load_4d(sA + stage * kABytes, &p.tmA[tp.map], &full[stage], kc * kBlockK, ow0 + tp.dw, oh0 + tp.dh, b);
            if (CLUSTER > 1)
              tma_load_3d_mc(sB + stage * B_BYTES + crank * (B_BYTES / 2), &p.tmBh, &full[stage], kc * kBlockK, tp.tap,
                             n0 + crank * (BLOCK_N / 2), static_cast<uint16_t>(0x3));
            else
              tma_load_3d(sB + stage * B_BYTES, &p.tmB, &full[stage], kc * kBlockK, tp.tap, n0);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp == 1) {
    // ---------------- epilogue DMA: lane 0 issues (and so owns the bulk-store groups it waits on), every lane copies columns
    const bool stage_y = EPI != kEpiF32 && (!ANY || p.y_dtype != UC_F32);
    const bool load_res = EPI == kEpiRes || EPI == kEpiReluRes || (ANY && p.res);
    for (int item = item0; item < num_items; item += item_step) {
      const int n0 = (item % p.n_tiles) * BLOCK_N;
      const int mt = (item / p.n_tiles) * CLUSTER + crank;
      const bool tile_ok = mt < p.m_tiles;
      const int ow0 = (mt % p.tiles_w) * p.tile_w, oh0 = ((mt / p.tiles_w) % p.tiles_h) * p.tile_h;
      const int b = mt / (p.tiles_w * p.tiles_h);
      const int limit = min(BLOCK_N, p.Cout - n0);
      const int nslabs = (limit + SLAB - 1) / SLAB;  // slabs holding valid columns
      // the consumers are done with the previous tile's slices (kEpiBar below); no 16-byte alignment is guaranteed here
      for (int i = lane; i < BLOCK_N; i += 32) {
        const bool in = i < limit;
        s_bias[i] = in && p.bias ? __ldg(p.bias + n0 + i) : 0.f;
        s_gamma[i] = in && p.gamma ? __ldg(p.gamma + n0 + i) : 1.f;  // x * 1 is exact: no branch on gamma in the epilogue
        if (use_ln) s_cols[i] = in ? __ldg(p.col_s + n0 + i) : 0.f;
      }
      if (lane == 0) {
        tma_store_wait_read();  // the previous tile's store has read the staging tile
        if (load_res && tile_ok) {
          mbar_arrive_expect_tx(epi_full, nslabs * SLAB_BYTES);
          for (int j = 0; j < nslabs; ++j) tma_load_4d(sY + j * SLAB_BYTES, &p.tmR, epi_full, n0 + j * SLAB, ow0, oh0, b);
        } else {
          mbar_arrive(epi_full);
        }
      } else {
        mbar_arrive(epi_full);
      }
      named_sync(kEpiBar, kConvConsumers * 128 + 32);  // the consumers have staged this tile
      if (stage_y && tile_ok && lane == 0) {
        for (int j = 0; j < nslabs; ++j) tma_store_4d(&p.tmY, sY + j * SLAB_BYTES, n0 + j * SLAB, ow0, oh0, b);
        tma_store_commit();
      }
    }
    if (lane == 0) tma_store_wait_all();
  } else if (wg > 0) {
    regs_alloc<232>();
    // ---------------- consumers: warpgroup c = pixels 64c .. 64c+63 of the tile.  Accumulator fragment of thread (warp w of the
    // warpgroup, lane = 4 g + t): rows r0 = 16 w + g and r0 + 8; registers 4i, 4i+1 = row r0, columns 8i + 2t, 8i + 2t + 1;
    // registers 4i+2, 4i+3 = row r0 + 8, same columns.
    const int c = wg - 1, ct = threadIdx.x - 128;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = c * 64 + (warp & 3) * 16 + g;
    const bool f16o = EPI == kEpiBiasF16 || (ANY && p.y_dtype == UC_F16);
    const bool f32o = EPI == kEpiF32 || (ANY && p.y_dtype == UC_F32);
    const bool has_res = EPI == kEpiRes || EPI == kEpiReluRes || (ANY && p.res != nullptr);
    const bool relu_res = EPI == kEpiReluRes || (ANY && p.relu_res);
    const bool use_gamma = EPI == kEpiRes || ANY;
    const int act = ANY ? p.act : EPI == kEpiRelu ? UC_ACT_RELU : (EPI == kEpiGelu || EPI == kEpiGeluLn) ? UC_ACT_GELU : UC_ACT_NONE;
    // GroupNorm: chunk i (columns 8i .. 8i+7) starts a new run of partial sums when a group boundary falls between its columns and
    // those of chunk i-1 (then some lane's group changed).  The same for every tile, and warp-uniform.
    uint32_t gn_new = 0;
    if (use_gn) {
  #pragma unroll 1
      for (int i = 1; i < BLOCK_N / 8; ++i) gn_new |= static_cast<uint32_t>((8 * i + 7) / p.gn_gs != (8 * i - 8) / p.gn_gs) << i;
    }
    // this thread's two staging rows: byte offset inside a slab, and the swizzle (16-byte chunk XOR) of the row
    uint32_t srow[2], sswz[2];
  #pragma unroll
    for (int h = 0; h < 2; ++h) {
      srow[h] = (r0 + 8 * h) * (SLAB * 2);
      sswz[h] = ((srow[h] >> 7) & (SLAB / 8 - 1)) << 4;
    }
    const uint64_t a_desc0 = wgmma_desc_sw128(smem_u32(sA + c * 64 * 128)), b_desc0 = wgmma_desc_sw128(smem_u32(sB));
    int stage = 0, phase = 0, gpar = 0, epar = 0;
    float acc[NACC];
    for (int item = item0; item < num_items; item += item_step) {
      const int n0 = (item % p.n_tiles) * BLOCK_N;
      const int mt = (item / p.n_tiles) * CLUSTER + crank;
      const bool tile_ok = mt < p.m_tiles;  // false: padding tile of an odd pair
      const int ow0 = (mt % p.tiles_w) * p.tile_w, oh0 = ((mt / p.tiles_w) % p.tiles_h) * p.tile_h;
      const int b = mt / (p.tiles_w * p.tiles_h);
      // ---- K loop: one wgmma group per stage in flight; a stage is released once the group after it has been issued
      int prev_stage = -1;
      for (int it = 0; it < kiters; ++it) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint64_t a_desc = a_desc0 + static_cast<uint64_t>((stage * kABytes) >> 4);
        const uint64_t b_desc = b_desc0 + static_cast<uint64_t>((stage * B_BYTES) >> 4);
  #pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) wgmma_ss<BLOCK_N, F16>(acc, a_desc + 2 * k, b_desc + 2 * k, (it | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev_stage >= 0 && ct % 128 == 0) release(prev_stage);
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev_stage >= 0 && ct % 128 == 0) release(prev_stage);

      // ---- epilogue straight from the accumulator registers
      const int limit = min(BLOCK_N, p.Cout - n0);  // valid columns of this tile (multiple of 8)
      size_t pix[2];
      bool valid[2];
      float r_rstd[2] = {1.f, 1.f}, r_murstd[2] = {0.f, 0.f};
  #pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        const int ow = ow0 + row % p.tile_w, oh = oh0 + row / p.tile_w;
        valid[h] = (ow < p.Wo) && (oh < p.Ho) && tile_ok;
        pix[h] = (static_cast<size_t>(b) * p.Ho + oh) * p.Wo + ow;
        // LayerNorm folded into the GEMM: y = rstd * (W' x) - rstd * mu * colsum(W') + c ; (mu, rstd) of this row's pixel
        if (use_ln && valid[h]) {  // fp32 is enough here (|mu| <~ 10 sigma for a ConvNeXt block's depthwise output)
          const longlong2 st = __ldg(reinterpret_cast<const longlong2*>(p.row_stats) + pix[h]);
          const float mu = static_cast<float>(st.x) * p.row_inv;
          const float var = fmaxf(fmaf(-mu, mu, static_cast<float>(st.y) * p.row_inv), 0.f);
          r_rstd[h] = rsqrtf(var + p.row_eps);
          r_murstd[h] = mu * r_rstd[h];
        }
      }
      // GroupNorm partial sums: per thread and column parity j, summed over the chunks of one run (gn_new), then over the 16 rows
      // of the warp (shuffles) and added to the CTA's shared-memory slots by lanes 0..3 (fixed point, integer adds: order
      // independent).  `cl` is a column of the run being flushed.
      unsigned long long* gacc = gn_acc + gpar * (kGnMaxLocal * 2);
      float gs1[2] = {0.f, 0.f}, gs2[2] = {0.f, 0.f};
      auto gn_flush = [&](int cl) {
  #pragma unroll
        for (int j = 0; j < 2; ++j) {
  #pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            gs1[j] += __shfl_xor_sync(0xffffffffu, gs1[j], o);
            gs2[j] += __shfl_xor_sync(0xffffffffu, gs2[j], o);
          }
          if (g == 0) {
            unsigned long long* slot = gacc + s_grp[cl + j] * 2;
            smem_add_u64(slot, static_cast<unsigned long long>(__float2ll_rn(gs1[j] * kGnFixedScale)));
            smem_add_u64(slot + 1, static_cast<unsigned long long>(__float2ll_rn(gs2[j] * kGnFixedScale)));
          }
          gs1[j] = gs2[j] = 0.f;
        }
      };
      mbar_wait(epi_full, epar);  // residual (staged in place of the output) and column slices of this tile
      epar ^= 1;
  #pragma unroll
      for (int i = 0; i < BLOCK_N / 8; ++i) {
        if (8 * i >= limit) break;  // warp-uniform
        const int cl = 8 * i + 2 * t;
        uint8_t* const slab = sY + (8 * i / SLAB) * SLAB_BYTES;
        const uint32_t cbyte = (8 * i % SLAB + 2 * t) * 2;
        const float2 bb = *reinterpret_cast<const float2*>(s_bias + cl);
        f32x2 hv[2];
  #pragma unroll
        for (int h = 0; h < 2; ++h) {
          const f32x2 v = pk2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
          if (use_ln) {
            const float2 cs = *reinterpret_cast<const float2*>(s_cols + cl);
            const f32x2 nm = pk2(-r_murstd[h], -r_murstd[h]);
            hv[h] = fma2(v, pk2(r_rstd[h], r_rstd[h]), fma2(nm, pk2(cs.x, cs.y), pk2(bb.x, bb.y)));
          } else {
            hv[h] = add2(v, pk2(bb.x, bb.y));
          }
        }
        if (use_gn) {
          if ((gn_new >> i) & 1u) gn_flush(cl - 8);
  #pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float x0 = valid[h] ? lo2(hv[h]) : 0.f, x1 = valid[h] ? hi2(hv[h]) : 0.f;
            gs1[0] += x0; gs2[0] = fmaf(x0, x0, gs2[0]);
            gs1[1] += x1; gs2[1] = fmaf(x1, x1, gs2[1]);
          }
        }
        if (act != UC_ACT_NONE) {
  #pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (act == UC_ACT_GELU) hv[h] = gelu2(hv[h]);
            else if (act == UC_ACT_RELU) hv[h] = pk2(fmaxf(lo2(hv[h]), 0.f), fmaxf(hi2(hv[h]), 0.f));
            else hv[h] = pk2(apply_act(lo2(hv[h]), act), apply_act(hi2(hv[h]), act));
          }
        }
        float2 gm = make_float2(1.f, 1.f);
        if (use_gamma) gm = *reinterpret_cast<const float2*>(s_gamma + cl);
  #pragma unroll
        for (int h = 0; h < 2; ++h) {
          // rounded product: a contraction with the residual add below into one FMA would change the result's bits
          if (use_gamma) hv[h] = pk2(__fmul_rn(lo2(hv[h]), gm.x), __fmul_rn(hi2(hv[h]), gm.y));
          if (f32o) {  // no residual with fp32 y
            if (valid[h]) *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.y) + pix[h] * p.ldy + n0 + cl) = hv[h];
            continue;
          }
          uint32_t* const sy = reinterpret_cast<uint32_t*>(slab + srow[h] + (cbyte ^ sswz[h]));
          if (has_res) {
            const uint32_t rw = *sy;
            hv[h] = add2(hv[h], f16o ? pk2(bits16_to_float(rw & 0xffffu, UC_F16), bits16_to_float(rw >> 16, UC_F16)) : pk2(bf16lo(rw), bf16hi(rw)));
          }
          if (relu_res) hv[h] = pk2(fmaxf(lo2(hv[h]), 0.f), fmaxf(hi2(hv[h]), 0.f));
          *sy = pack2_fast(lo2(hv[h]), hi2(hv[h]), f16o);
        }
      }
      if (!f32o) fence_proxy_async();  // the TMA store (async proxy) reads what these generic-proxy writes staged
      named_arrive(kEpiBar, kConvConsumers * 128 + 32);
      if (use_gn) {
        gn_flush(((limit - 1) & ~7) + 2 * t);  // the run of the last chunk
        // every consumer thread has added its partial sums of this tile: one global atomic per group, then the slots are cleared for
        // the tile after next (the next tile uses the other parity, so no second barrier is needed)
        named_sync(1, kConvConsumers * 128);
        const int ng = (limit + p.gn_gs - 1) / p.gn_gs;
        if (ct < 2 * ng) {
          unsigned long long* slot = gacc + ct;
          const unsigned long long v = *slot;
          *slot = 0ull;
          if (tile_ok && v != 0ull) {
            unsigned long long* dst = reinterpret_cast<unsigned long long*>(p.gn_stats) + (static_cast<size_t>(b) * p.gn_groups + n0 / p.gn_gs) * 2 + ct;
            atomicAdd(dst, v);
          }
        }
        gpar ^= 1;
      }
    }
  }
  if (CLUSTER > 1) cluster_sync_all();  // no CTA exits while its peer can still multicast into it or arrive on its barriers
}

// ------------------------------------------------------------------------------------------- host side

template <int BLOCK_N, int STAGES, int CLUSTER, int EPI, bool F16>
static int launch_conv(const ConvKernelParams& p, cudaStream_t stream) {
  constexpr int smem = conv_smem_bytes(BLOCK_N, STAGES);
  static_assert(smem <= 227 * 1024, "conv_gemm: shared memory over the 227 KB per-block limit");
  static PerDeviceFlag attr_dev;
  bool& attr = attr_dev.get();
  auto kern = conv_gemm_kernel<BLOCK_N, STAGES, F16, CLUSTER, EPI>;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return set_error(static_cast<int>(e), "conv_gemm: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr = true;
  }
  const int items = p.n_tiles * ((p.m_tiles + CLUSTER - 1) / CLUSTER);
  int grid = std::min(items * CLUSTER, num_sms());  // one CTA per SM
  grid -= grid % CLUSTER;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kConvThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr_list[2];
  int na = 0;
  if (pdl_enabled()) {
    attr_list[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr_list[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (CLUSTER > 1) {
    attr_list[na].id = cudaLaunchAttributeClusterDimension;
    attr_list[na].val.clusterDim.x = CLUSTER;
    attr_list[na].val.clusterDim.y = 1;
    attr_list[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr_list;
  cfg.numAttrs = na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, p);
  if (e != cudaSuccess) return set_error(static_cast<int>(e), "conv_gemm<%d,%d,%d,%d> launch: %s", BLOCK_N, STAGES, CLUSTER, EPI, cudaGetErrorString(e));
  return UC_OK;
}

// Launches the instantiation of epilogue variant EPI (operands f16 if F16, else bf16) for N tile bn.  Each conv_gemm_*.cu file
// instantiates some of these; conv_gemm.cu calls them.
template <int EPI, bool F16>
int conv_launch(const ConvKernelParams& p, int bn, bool cluster2, cudaStream_t stream) {
  if (cluster2) {
    switch (bn) {
      case 256: return launch_conv<256, 3, 2, EPI, F16>(p, stream);
      case 192: return launch_conv<192, 4, 2, EPI, F16>(p, stream);
      case 128: return launch_conv<128, 5, 2, EPI, F16>(p, stream);
      default: return set_error(UC_EINVAL, "uc_conv2d: the cluster variant exists for block_n 128/192/256 only");
    }
  }
  switch (bn) {  // stage ring + output staging tile: 151 - 214 KB (227 KB of shared memory per block)
    case 256: return launch_conv<256, 3, 1, EPI, F16>(p, stream);
    case 192: return launch_conv<192, 4, 1, EPI, F16>(p, stream);
    case 128: return launch_conv<128, 5, 1, EPI, F16>(p, stream);
    case 96: return launch_conv<96, 6, 1, EPI, F16>(p, stream);
    case 64: return launch_conv<64, 8, 1, EPI, F16>(p, stream);
    case 32: return launch_conv<32, 8, 1, EPI, F16>(p, stream);
    case 16: return launch_conv<16, 8, 1, EPI, F16>(p, stream);
    default: return set_error(UC_EINVAL, "uc_conv2d: unsupported block_n %d", bn);
  }
}

#define UC_CONV_EPI_LIST(X) \
  X(kEpiAny, false) X(kEpiAny, true) X(kEpiBias, false) X(kEpiBiasF16, false) X(kEpiF32, false) X(kEpiRelu, false) \
  X(kEpiGelu, false) X(kEpiGeluLn, false) X(kEpiRes, false) X(kEpiReluRes, false) X(kEpiGn, false)
#define UC_CONV_EPI_EXTERN(E, F) extern template int conv_launch<E, F>(const ConvKernelParams&, int, bool, cudaStream_t);
UC_CONV_EPI_LIST(UC_CONV_EPI_EXTERN)
#undef UC_CONV_EPI_EXTERN

}  // namespace uc
