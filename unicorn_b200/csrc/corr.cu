// Fused reference<->current embedding correlation + softmax over reference positions + label propagation.
//
//   out[o, j] = sum_i V[o, i] * softmax_i( <K_i, Q_j> )        K = reference embedding, Q = current embedding
//
// replaces the three materialising passes of external/lib/test/tracker/unicorn_sot.py:95-100
// (torch.mm -> softmax(dim=0) -> values @ trans_mat; same in unicorn_vos.py:171-181): the (N_ref x N_cur) similarity
// matrix (512 MB in fp16 at 800x1280) never leaves the SM.  Flash-attention style: one CTA owns 128 current positions,
// streams the reference positions in chunks of 128 through a TMA ring, and each of two consumer warpgroups computes the
// 64 x 128 similarity tile of its 64 positions with wgmma (m64n128k16) into registers and keeps, per thread, the running
// max / sum / weighted label sums of the columns it holds (no cross-thread reductions inside the loop; the four partial
// states of a position are merged once at the end).  One exponential in four is evaluated on the FMA pipe (the softmax is
// bound by the MUFU unit).  V has only n_obj (1..8) rows, so the P.V product is done with CUDA-core FMAs on the
// probabilities instead of wasting an MMA tile.
#include "uc_ptx.cuh"
#include "uc_common.h"
#include "../../include/unicorn_b200.h"

namespace uc {

constexpr int kCorrC = 128;       // embedding channels
constexpr int kCorrTile = 128;    // current positions per CTA (64 per consumer warpgroup)
constexpr int kCorrChunk = 128;   // reference positions per MMA chunk (64 accumulator registers per thread)
constexpr int kCorrStages = 4;    // K ring (32 KB per stage; the chunk's label values travel with it)
constexpr int kCorrQBytes = kCorrTile * kCorrC * 2;    // 32 KB (two 128B-swizzled 64-channel halves)
constexpr int kCorrKBytes = kCorrChunk * kCorrC * 2;   // 32 KB
constexpr int kCorrConsumers = 2;
constexpr int kCorrThreads = (1 + kCorrConsumers) * 128;

struct alignas(64) CorrParams {
  CUtensorMap tmQ, tmK;  // [B][n][C]
  const float* V;  // [B][n_obj, ldv], sequence stride bsv
  float* out;      // [B][n_obj, ldo], sequence stride bso
  long bsv, bso;
  int ldv, ldo, n_cur, n_ref, n_obj;
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 2^x for x <= 0 on the FMA / ALU pipes (no MUFU): round-to-nearest split x = n + f, |f| <= 0.5, 2^f by a degree-4 minimax polynomial
// (max relative error 2.9e-6 — below the bf16/fp16 rounding of the similarity itself), 2^n by an exponent-field add.  One element in
// four takes this path: the kernel is bound by the MUFU unit (16 ex2 per clock per SM), the FMA pipe has room for ~25 % of them.
__device__ __forceinline__ float poly_exp2(float x) {
  x = fmaxf(x, -125.f);
  const float t = x + 12582912.f;              // 1.5 * 2^23: the integer part lands in the low mantissa bits
  const float f = x - (t - 12582912.f);        // in [-0.5, 0.5]
  float p = fmaf(f, 9.582853e-3f, 5.5906426e-2f);  // weighted least-squares (near-minimax) fit on [-0.5, 0.5] with p(0) = 1
  p = fmaf(p, f, 2.4024099e-1f);
  p = fmaf(p, f, 6.9312418e-1f);
  p = fmaf(p, f, 1.f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}

template <int NOBJ, bool F16>
__global__ void __launch_bounds__(kCorrThreads, 1) corr_kernel(const __grid_constant__ CorrParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sK = smem + kCorrQBytes;
  float* sV = reinterpret_cast<float*>(sK + kCorrStages * kCorrKBytes);  // [kCorrStages][NOBJ][kCorrChunk]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sV + kCorrStages * NOBJ * kCorrChunk);
  uint64_t* k_full = q_full + 1;
  uint64_t* k_empty = k_full + kCorrStages;

  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j0 = blockIdx.x * kCorrTile;
  const int seq = blockIdx.y;  // one (reference, current, values) triple per grid row
  const float* const V = p.V + seq * p.bsv;
  const int nchunks = (p.n_ref + kCorrChunk - 1) / kCorrChunk;

  if (threadIdx.x == 0) {
    prefetch_tmap(&p.tmQ);
    prefetch_tmap(&p.tmK);
    mbar_init(q_full, 1);
    // full: TMA bytes + label values; empty: one arrival per consumer WARP (every warp reads the stage's label values itself)
    for (int i = 0; i < kCorrStages; ++i) { mbar_init(&k_full[i], 2); mbar_init(&k_empty[i], kCorrConsumers * 4); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();  // barrier init above overlapped the previous kernel's tail
  pdl_launch_dependents();

  if (wg == 0) {
    if (warp != 0) return;
    // Producer: TMA for the K chunk (one elected lane) and — all 32 lanes — the chunk's label values V[:, i0 .. i0+127] into the
    // same stage.  The producer runs up to kCorrStages chunks ahead, so the L2 latency of these loads is off the softmax's path.
    if (elect_one()) {
      mbar_arrive_expect_tx(q_full, kCorrQBytes);
      tma_load_3d(sQ, &p.tmQ, q_full, 0, j0, seq);
      tma_load_3d(sQ + kCorrQBytes / 2, &p.tmQ, q_full, 64, j0, seq);
    }
    __syncwarp();
    int stage = 0, phase = 0;
    for (int c = 0; c < nchunks; ++c) {
      mbar_wait(&k_empty[stage], phase ^ 1);
      const int i0 = c * kCorrChunk;
      if (elect_one()) {
        mbar_arrive_expect_tx(&k_full[stage], kCorrKBytes);
        uint8_t* dst = sK + stage * kCorrKBytes;
        tma_load_3d(dst, &p.tmK, &k_full[stage], 0, i0, seq);
        tma_load_3d(dst + kCorrKBytes / 2, &p.tmK, &k_full[stage], 64, i0, seq);
      }
      float* vb = sV + stage * NOBJ * kCorrChunk;
#pragma unroll
      for (int o = 0; o < NOBJ; ++o) {
#pragma unroll
        for (int t = 0; t < kCorrChunk / 32; ++t) {
          const int i = i0 + t * 32 + lane;
          vb[o * kCorrChunk + t * 32 + lane] = (o < p.n_obj && i < p.n_ref) ? __ldg(V + static_cast<long>(o) * p.ldv + i) : 0.f;
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_full[stage]);  // release: the consumers acquire it with their wait
      if (++stage == kCorrStages) { stage = 0; phase ^= 1; }
    }
    return;
  }
  // ---------------- consumers: S = Q K^T, online softmax + label propagation.  Warpgroup c owns positions 64c .. 64c+63;
  // thread (warp w, lane = 4 g + t) holds rows 16 w + g (h = 0) and + 8 (h = 1), columns 8i + 2t, 8i + 2t + 1 of the chunk.
  // Everything is in the log2 domain: p = 2^(s*log2e - m).
  const int c = wg - 1;
  const int g = lane >> 2, t = lane & 3;
  constexpr float kLog2e = 1.4426950408889634f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float acc[2][NOBJ];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int o = 0; o < NOBJ; ++o) acc[h][o] = 0.f;
  mbar_wait(q_full, 0);
  const uint64_t q_desc = wgmma_desc_sw128(smem_u32(sQ + c * 64 * 128)), k_desc0 = wgmma_desc_sw128(smem_u32(sK));
  int stage = 0, phase = 0;
  for (int cc = 0; cc < nchunks; ++cc) {
    const int i0 = cc * kCorrChunk;
    mbar_wait(&k_full[stage], phase);
    float s[kCorrChunk / 2];
    wgmma_fence();
    const uint64_t k_desc = k_desc0 + static_cast<uint64_t>((stage * kCorrKBytes) >> 4);
#pragma unroll
    for (int ks = 0; ks < kCorrC / 16; ++ks) {
      const uint64_t qo = static_cast<uint64_t>(((ks >> 2) * (kCorrQBytes / 2) + (ks & 3) * 32) >> 4);
      const uint64_t ko = static_cast<uint64_t>(((ks >> 2) * (kCorrKBytes / 2) + (ks & 3) * 32) >> 4);
      wgmma_ss<kCorrChunk, F16>(s, q_desc + qo, k_desc + ko, ks != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    const int nvalid = min(kCorrChunk, p.n_ref - i0);
    if (nvalid < kCorrChunk) {  // tail chunk only (uniform)
#pragma unroll
      for (int i = 0; i < kCorrChunk / 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (8 * i + 2 * t + (e & 1) >= nvalid) s[4 * i + e] = -INFINITY;
    }
    const float* vb = sV + stage * NOBJ * kCorrChunk;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};  // tree maximum: no 32-deep dependent chain
#pragma unroll
      for (int i = 0; i < kCorrChunk / 8; ++i) mx[i & 3] = fmaxf(mx[i & 3], fmaxf(s[4 * i + 2 * h], s[4 * i + 2 * h + 1]));
      const float cmax = fmaxf(fmaxf(mx[0], mx[1]), fmaxf(mx[2], mx[3]));
      if (cmax == -INFINITY) continue;  // every column of this thread is masked (tail chunk)
      const float m_new = fmaxf(m[h], cmax * kLog2e);
      if (m_new != m[h]) {  // the running maximum moves in the first few chunks only: skip the rescale otherwise
        const float scale = fast_exp2(m[h] - m_new);
        m[h] = m_new;
        l[h] *= scale;
#pragma unroll
        for (int o = 0; o < NOBJ; ++o) acc[h][o] *= scale;
      }
      const float neg_m = -m_new;
#pragma unroll
      for (int i = 0; i < kCorrChunk / 8; ++i) {
        const float x0 = fmaf(s[4 * i + 2 * h], kLog2e, neg_m), x1 = fmaf(s[4 * i + 2 * h + 1], kLog2e, neg_m);  // <= 0
        const float p0 = fast_exp2(x0), p1 = (i & 1) ? poly_exp2(x1) : fast_exp2(x1);
        l[h] += p0 + p1;
#pragma unroll
        for (int o = 0; o < NOBJ; ++o) {
          const float2 vv = *reinterpret_cast<const float2*>(vb + o * kCorrChunk + 8 * i + 2 * t);
          acc[h][o] = fmaf(p1, vv.y, fmaf(p0, vv.x, acc[h][o]));
        }
      }
    }
    // K chunk and label values of this stage consumed by this warp: the label values are read with ordinary loads by every lane, so
    // the slot may be refilled only when all lanes of all consumer warps are past their last read (a per-warpgroup release from one
    // thread would not order the other warps' reads)
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[stage]);
    if (++stage == kCorrStages) { stage = 0; phase ^= 1; }
  }
  // merge the four partial states of every position (the 4 lanes t of a quad)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float M = m[h];
    M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 1));
    M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 2));
    const float w = fast_exp2(m[h] - M);  // a thread that saw only masked columns has m = -inf -> weight 0
    float L = l[h] * w;
    L += __shfl_xor_sync(0xffffffffu, L, 1);
    L += __shfl_xor_sync(0xffffffffu, L, 2);
    float A[NOBJ];
#pragma unroll
    for (int o = 0; o < NOBJ; ++o) {
      A[o] = acc[h][o] * w;
      A[o] += __shfl_xor_sync(0xffffffffu, A[o], 1);
      A[o] += __shfl_xor_sync(0xffffffffu, A[o], 2);
    }
    const int j = j0 + c * 64 + (warp & 3) * 16 + g + 8 * h;
    if (t == 0 && j < p.n_cur) {
      const float inv = 1.f / L;
#pragma unroll
      for (int o = 0; o < NOBJ; ++o)
        if (o < p.n_obj) p.out[seq * p.bso + static_cast<long>(o) * p.ldo + j] = A[o] * inv;
    }
  }
}

template <int NOBJ>
static int launch_corr(const CorrParams& p, bool f16, dim3 grid, const char* what, cudaStream_t stream) {
  constexpr int smem = kCorrQBytes + kCorrStages * kCorrKBytes + kCorrStages * NOBJ * kCorrChunk * 4 + 256 + 1024;
  static PerDeviceFlag attr_dev;
  bool& attr_set = attr_dev.get();
  if (!attr_set) {
    for (auto k : {corr_kernel<NOBJ, true>, corr_kernel<NOBJ, false>}) {
      cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      if (e != cudaSuccess) return set_error(static_cast<int>(e), "corr: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    }
    attr_set = true;
  }
  launch_pdl(f16 ? corr_kernel<NOBJ, true> : corr_kernel<NOBJ, false>, grid, kCorrThreads, smem, stream, p);
  return check_launch(what);
}

// B (reference, current, values) triples; the strides bs_* between sequences are in elements.  B = 1 ignores them.
static int corr_propagate(const char* what, const void* embed_ref, int ld_ref, long bs_ref, int n_ref, const void* embed_cur, int ld_cur,
                          long bs_cur, int n_cur, int C, int dtype, const float* values, int ldv, long bs_v, int n_obj, float* out,
                          int ldo, long bs_out, int B, void* stream_v) {
  if (!embed_ref || !embed_cur || !values || !out) return set_error(UC_EINVAL, "%s: null pointer", what);
  if (B < 1) return set_error(UC_EINVAL, "%s: B must be >= 1 (got %d)", what, B);
  if (C != kCorrC) return set_error(UC_EINVAL, "%s: embedding dim must be %d (got %d)", what, kCorrC, C);
  if (dtype != UC_BF16 && dtype != UC_F16) return set_error(UC_EINVAL, "%s: embeddings must be bf16/f16", what);
  if (n_obj < 1 || n_obj > 8) return set_error(UC_EINVAL, "%s: 1 <= n_obj <= 8 (got %d)", what, n_obj);
  if (ld_ref % 8 || ld_cur % 8 || n_ref < 1 || n_cur < 1 || ldv < n_ref || ldo < n_cur) return set_error(UC_EINVAL, "%s: bad sizes/strides", what);
  if (B == 1) {
    bs_ref = static_cast<long>(ld_ref) * n_ref; bs_cur = static_cast<long>(ld_cur) * n_cur;
    bs_v = static_cast<long>(ldv) * n_obj; bs_out = static_cast<long>(ldo) * n_obj;
  } else if (bs_ref % 8 || bs_cur % 8 || bs_ref < static_cast<long>(ld_ref) * n_ref || bs_cur < static_cast<long>(ld_cur) * n_cur ||
             bs_v < static_cast<long>(ldv) * n_obj || bs_out < static_cast<long>(ldo) * n_obj) {
    return set_error(UC_EINVAL, "%s: bad per-sequence strides (embeddings: multiple of 8 and >= ld*n; values / out: >= ld*n_obj)", what);
  }
  int rc = ensure_driver();
  if (rc) return rc;
  CorrParams p;
  memset(&p, 0, sizeof(p));
  const CUtensorMapDataType dt = dtype == UC_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  {
    uint64_t dims[3] = {static_cast<uint64_t>(C), static_cast<uint64_t>(n_cur), static_cast<uint64_t>(B)};
    uint64_t strides[2] = {static_cast<uint64_t>(ld_cur) * 2, static_cast<uint64_t>(bs_cur) * 2};
    uint32_t box[3] = {64, kCorrTile, 1};
    rc = encode_tmap(&p.tmQ, dt, 3, embed_cur, dims, strides, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {static_cast<uint64_t>(C), static_cast<uint64_t>(n_ref), static_cast<uint64_t>(B)};
    uint64_t strides[2] = {static_cast<uint64_t>(ld_ref) * 2, static_cast<uint64_t>(bs_ref) * 2};
    uint32_t box[3] = {64, kCorrChunk, 1};
    rc = encode_tmap(&p.tmK, dt, 3, embed_ref, dims, strides, box);
    if (rc) return rc;
  }
  p.V = values; p.out = out; p.bsv = bs_v; p.bso = bs_out;
  p.ldv = ldv; p.ldo = ldo; p.n_cur = n_cur; p.n_ref = n_ref; p.n_obj = n_obj;
  const bool f16 = dtype == UC_F16;
  const dim3 grid((n_cur + kCorrTile - 1) / kCorrTile, B);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_obj == 1) return launch_corr<1>(p, f16, grid, what, stream);
  if (n_obj == 2) return launch_corr<2>(p, f16, grid, what, stream);
  if (n_obj <= 4) return launch_corr<4>(p, f16, grid, what, stream);
  return launch_corr<8>(p, f16, grid, what, stream);
}

}  // namespace uc

using namespace uc;

extern "C" int uc_corr_propagate(const void* embed_ref, int ld_ref, int n_ref, const void* embed_cur, int ld_cur, int n_cur,
                                 int C, int dtype, const float* values, int ldv, int n_obj, float* out, int ldo,
                                 void* stream_v) {
  return corr_propagate("uc_corr_propagate", embed_ref, ld_ref, 0, n_ref, embed_cur, ld_cur, 0, n_cur, C, dtype, values, ldv, 0, n_obj,
                        out, ldo, 0, 1, stream_v);
}

extern "C" int uc_corr_propagate_batched(const void* embed_ref, int ld_ref, long bs_ref, int n_ref, const void* embed_cur, int ld_cur,
                                         long bs_cur, int n_cur, int C, int dtype, const float* values, int ldv, long bs_values,
                                         int n_obj, float* out, int ldo, long bs_out, int B, void* stream_v) {
  return corr_propagate("uc_corr_propagate_batched", embed_ref, ld_ref, bs_ref, n_ref, embed_cur, ld_cur, bs_cur, n_cur, C, dtype, values,
                        ldv, bs_values, n_obj, out, ldo, bs_out, B, stream_v);
}
