// Detection post-processing on the device: head decode, score filter, sort, class-aware NMS.
//   uc_head_decode   unicorn_head.py:332-334 (cat[reg, sigmoid(obj), sigmoid(cls)]) + decode_outputs :467-482
//   uc_postprocess   unicorn/utils/boxes.py:33-77: cxcywh->xyxy, class_conf/pred = max/argmax over classes,
//                    keep obj*class_conf >= conf, torchvision.ops.batched_nms (greedy, IoU > thr suppresses,
//                    only within the same class), result ordered by descending score.
//   uc_det_candidates_batched   the decode + filter of the two above fused, read straight from the per-level head maps
//   UC_POST_CLASS_AGNOSTIC      postprocess(..., class_agnostic=True): torchvision.ops.nms over all classes
// Everything stays on the GPU; the host reads back one counter.  Decision arithmetic is fp32 with the reference's roundings:
// the score filter is rn(obj * class_conf) >= conf (first maximum over classes), and NMS is torchvision's CUDA devIoU with
// the later box's area fused into the union (nms_hit), so kept sets, order and count equal torchvision.ops.nms on CUDA
// bit for bit (class-aware: per class), equal scores kept in ascending candidate order.  Not matched: torchvision's CPU nms,
// which compares in double, and the class offsets batched_nms adds on CUDA up to 5000 boxes, which re-round the IoU.
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include <algorithm>

namespace uc {

struct DecodeLevels {
  const float* regobj[3];  // [B][HW, ld_ro]: reg(4), obj logit
  const float* cls[3];     // [B][HW, ld_cls]: class logits
  long bs_ro[3], bs_cls[3];  // per-level image strides (elements)
  int h[3], w[3], stride[3], start[3];
  int ld_ro, ld_cls, ncls, total;
};

__global__ void __launch_bounds__(256) head_decode_kernel(DecodeLevels lv, float* __restrict__ out) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;  // image
  if (i >= lv.total) return;
  int k = 0;
  if (i >= lv.start[1]) k = 1;
  if (i >= lv.start[2]) k = 2;
  const int a = i - lv.start[k];
  const int x = a % lv.w[k], y = a / lv.w[k];
  const float s = static_cast<float>(lv.stride[k]);
  const float* ro = lv.regobj[k] + b * lv.bs_ro[k] + static_cast<long>(a) * lv.ld_ro;
  const float* cl = lv.cls[k] + b * lv.bs_cls[k] + static_cast<long>(a) * lv.ld_cls;
  float* o = out + (static_cast<long>(b) * lv.total + i) * (5 + lv.ncls);
  o[0] = (ro[0] + x) * s;
  o[1] = (ro[1] + y) * s;
  o[2] = expf(ro[2]) * s;
  o[3] = expf(ro[3]) * s;
  o[4] = 1.f / (1.f + expf(-ro[4]));
  for (int c = 0; c < lv.ncls; ++c) o[5 + c] = 1.f / (1.f + expf(-cl[c]));
}

// Per-image slices of the postprocess workspace: image b owns bytes [b * per_image, (b + 1) * per_image), laid out as
// count (256 bytes), det [A][7], sorted [A][7] (fp32), keys [a2] (u64), det_anchor [A], sorted_anchor [A] (int).
struct PostSlices {
  uint8_t* ws;
  long per_image, a2;
  int A;
  __device__ __forceinline__ uint8_t* base(int b) const { return ws + b * per_image; }
  __device__ __forceinline__ int* count(int b) const { return reinterpret_cast<int*>(base(b)); }
  // per-tile candidate counts of det_candidates (the rest of the 256-byte count header)
  __device__ __forceinline__ int* tile_count(int b) const { return count(b) + 1; }
  __device__ __forceinline__ float* det(int b) const { return reinterpret_cast<float*>(base(b) + 256); }
  __device__ __forceinline__ float* sorted(int b) const { return det(b) + static_cast<long>(A) * 7; }
  __device__ __forceinline__ unsigned long long* keys(int b) const {
    return reinterpret_cast<unsigned long long*>(sorted(b) + static_cast<long>(A) * 7);
  }
  __device__ __forceinline__ int* det_anchor(int b) const { return reinterpret_cast<int*>(keys(b) + a2); }
  __device__ __forceinline__ int* sorted_anchor(int b) const { return det_anchor(b) + A; }
};

// ---- filter: deterministic compaction (anchor order) of candidates with obj*class_conf >= conf.
// det rows: x1,y1,x2,y2,obj,class_conf,class_pred ; key = (score bits << 32) | (0xffffffff - candidate index)
__global__ void __launch_bounds__(1024) det_filter_kernel(const float* __restrict__ pred, int A, int ncls, float conf, PostSlices sl) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int cap = A;
  pred += static_cast<long>(blockIdx.x) * A * (5 + ncls);
  float* const det = sl.det(blockIdx.x);
  unsigned long long* const keys = sl.keys(blockIdx.x);
  int* const count = sl.count(blockIdx.x);
  int* const det_anchor = sl.det_anchor(blockIdx.x);
  __shared__ int warp_cnt[32];
  __shared__ int warp_excl[32];
  __shared__ int base, round_total;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int a0 = 0; a0 < A; a0 += 1024) {
    const int a = a0 + threadIdx.x;
    bool pass = false;
    float r[7];
    float score = 0.f;
    if (a < A) {
      const float* p = pred + static_cast<long>(a) * (5 + ncls);
      float best = p[5];
      int bi = 0;
      for (int c = 1; c < ncls; ++c) {
        const float v = p[5 + c];
        if (v > best) { best = v; bi = c; }
      }
      score = p[4] * best;
      pass = score >= conf;
      r[0] = p[0] - p[2] / 2; r[1] = p[1] - p[3] / 2; r[2] = p[0] + p[2] / 2; r[3] = p[1] + p[3] / 2;
      r[4] = p[4]; r[5] = best; r[6] = static_cast<float>(bi);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, pass);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    if (warp == 0) {
      const int v = warp_cnt[lane];
      int incl = v;
      for (int o = 1; o < 32; o <<= 1) {
        const int nb = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += nb;
      }
      warp_excl[lane] = incl - v;
      if (lane == 31) round_total = incl;
    }
    __syncthreads();
    if (pass) {
      const int idx = base + warp_excl[warp] + __popc(bal & ((1u << lane) - 1));
      if (idx < cap) {
        float* d = det + static_cast<long>(idx) * 7;
#pragma unroll
        for (int t = 0; t < 7; ++t) d[t] = r[t];
        keys[idx] = (static_cast<unsigned long long>(__float_as_uint(score)) << 32) | (0xffffffffu - static_cast<unsigned>(idx));
        det_anchor[idx] = a;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) base += round_total;
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = min(base, cap);
}

// ---- fused decode + filter for wide heads, straight from the per-level maps (head_decode + det_filter without the [B, A, 5+ncls]
// tensor in between).  Same fp32 operations in the same order as those two kernels (the _rn intrinsics keep nvcc from contracting
// the decode's product into the corner's sum, which the stored intermediate prevents there), so rows, keys, anchor ids and counts
// are bit-identical.  Two launches per image, each on ntiles CTAs:
//   1. every CTA takes a tile of anchors, compacts its candidates in anchor order into its own region of the `sorted` rows /
//      `sorted_anchor` (both free until the gather) and writes its candidate count into the slice header;
//   2. every CTA sums the counts of the tiles before its own and copies its candidates to their final place, with their keys.
constexpr int kCandThreads = 256;
constexpr int kCandMaxTiles = 63;  // tile counts live in the 256-byte header after the count

static int cand_tile(int A) {  // anchors per tile: a multiple of the CTA size, at most kCandMaxTiles tiles
  const int per = (A + kCandMaxTiles - 1) / kCandMaxTiles;
  return std::max(1, (per + kCandThreads - 1) / kCandThreads) * kCandThreads;
}

__global__ void __launch_bounds__(kCandThreads) det_candidates_kernel(DecodeLevels lv, int tile, float conf, PostSlices sl) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y, t0 = blockIdx.x * tile;
  float* const stage = sl.sorted(b) + static_cast<long>(t0) * 7;
  int* const stage_anchor = sl.sorted_anchor(b) + t0;
  __shared__ int warp_cnt[kCandThreads / 32];
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int end = min(t0 + tile, lv.total);
  for (int a0 = t0; a0 < end; a0 += kCandThreads) {
    const int i = a0 + threadIdx.x;
    bool pass = false;
    float r[7];
    if (i < end) {
      int k = 0;
      if (i >= lv.start[1]) k = 1;
      if (i >= lv.start[2]) k = 2;
      const int a = i - lv.start[k];
      const float x = static_cast<float>(a % lv.w[k]), y = static_cast<float>(a / lv.w[k]);
      const float s = static_cast<float>(lv.stride[k]);
      const float* ro = lv.regobj[k] + b * lv.bs_ro[k] + static_cast<long>(a) * lv.ld_ro;
      const float* cl = lv.cls[k] + b * lv.bs_cls[k] + static_cast<long>(a) * lv.ld_cls;
      const float cx = __fmul_rn(__fadd_rn(ro[0], x), s), cy = __fmul_rn(__fadd_rn(ro[1], y), s);
      const float w = __fmul_rn(expf(ro[2]), s), h = __fmul_rn(expf(ro[3]), s);
      const float obj = 1.f / (1.f + expf(-ro[4]));
      float best = 1.f / (1.f + expf(-cl[0]));
      int bi = 0;
      for (int c = 1; c < lv.ncls; ++c) {  // compared after the sigmoid: saturated logits tie and the first class wins, as in torch.max
        const float v = 1.f / (1.f + expf(-cl[c]));
        if (v > best) { best = v; bi = c; }
      }
      pass = __fmul_rn(obj, best) >= conf;
      r[0] = __fsub_rn(cx, __fmul_rn(w, 0.5f)); r[1] = __fsub_rn(cy, __fmul_rn(h, 0.5f));
      r[2] = __fadd_rn(cx, __fmul_rn(w, 0.5f)); r[3] = __fadd_rn(cy, __fmul_rn(h, 0.5f));
      r[4] = obj; r[5] = best; r[6] = static_cast<float>(bi);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, pass);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    if (pass) {
      int idx = base + __popc(bal & ((1u << lane) - 1));
      for (int q = 0; q < warp; ++q) idx += warp_cnt[q];
      float* d = stage + static_cast<long>(idx) * 7;
#pragma unroll
      for (int q = 0; q < 7; ++q) d[q] = r[q];
      stage_anchor[idx] = i;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int n = 0;
      for (int q = 0; q < kCandThreads / 32; ++q) n += warp_cnt[q];
      base += n;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) sl.tile_count(b)[blockIdx.x] = base;
}

__global__ void __launch_bounds__(kCandThreads) det_candidates_compact_kernel(int tile, PostSlices sl) {
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.y, t = blockIdx.x;
  const int* const tc = sl.tile_count(b);
  __shared__ int off_s;
  if (threadIdx.x < 32) {
    int v = 0;
    for (int q = threadIdx.x; q < t; q += 32) v += tc[q];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) off_s = v;
  }
  __syncthreads();
  const int off = off_s, n = tc[t];
  const float* const stage = sl.sorted(b) + static_cast<long>(t) * tile * 7;
  const int* const stage_anchor = sl.sorted_anchor(b) + static_cast<long>(t) * tile;
  float* const det = sl.det(b);
  unsigned long long* const keys = sl.keys(b);
  int* const det_anchor = sl.det_anchor(b);
  for (int j = threadIdx.x; j < n; j += kCandThreads) {
    const float* src = stage + static_cast<long>(j) * 7;
    const int idx = off + j;
    float* d = det + static_cast<long>(idx) * 7;
#pragma unroll
    for (int q = 0; q < 7; ++q) d[q] = src[q];
    const float score = __fmul_rn(src[4], src[5]);
    keys[idx] = (static_cast<unsigned long long>(__float_as_uint(score)) << 32) | (0xffffffffu - static_cast<unsigned>(idx));
    det_anchor[idx] = stage_anchor[j];
  }
  if (t == gridDim.x - 1 && threadIdx.x == 0) *sl.count(b) = off + n;
}

// ---- sort keys descending (bitonic, one CTA per image, n2 = power of two >= count; pads with 0 keys)
__global__ void __launch_bounds__(1024) sort_desc_kernel(PostSlices sl) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  unsigned long long* const keys = sl.keys(blockIdx.x);
  const int* const count = sl.count(blockIdx.x);
  const int cap2 = static_cast<int>(sl.a2);
  const int n = *count;
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  if (n2 > cap2) n2 = cap2;
  for (int i = n + threadIdx.x; i < n2; i += blockDim.x) keys[i] = 0ull;
  __syncthreads();
  for (int k = 2; k <= n2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (n2 >> 1); t += blockDim.x) {
        const int i = ((t / j) * (j << 1)) + (t % j);
        const int ixj = i + j;
        const unsigned long long a = keys[i], b = keys[ixj];
        const bool desc = ((i & k) == 0);
        if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
      }
      __syncthreads();
    }
  }
}

// ---- gather rows in sorted order
__global__ void __launch_bounds__(256) det_gather_kernel(PostSlices sl) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int img = blockIdx.y;
  const float* const det = sl.det(img);
  const unsigned long long* const keys = sl.keys(img);
  const int* const count = sl.count(img);
  float* const sorted = sl.sorted(img);
  const int* const det_anchor = sl.det_anchor(img);
  int* const sorted_anchor = sl.sorted_anchor(img);
  const int n = *count;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned idx = 0xffffffffu - static_cast<unsigned>(keys[i] & 0xffffffffull);
    sorted_anchor[i] = det_anchor[idx];
#pragma unroll
    for (int t = 0; t < 7; ++t) sorted[static_cast<long>(i) * 7 + t] = det[static_cast<long>(idx) * 7 + t];
  }
}

// ---- greedy NMS without an N x N matrix (one CTA).  Candidates are visited in score order in chunks of 256:
//  1. every candidate of the chunk is tested against the boxes kept so far (4 threads per candidate split the list);
//  2. the survivors of the chunk are tested against each other (256 x 256 bits in shared memory);
//  3. one warp resolves the chunk greedily, jumping from survivor to survivor with ffs;
//  4. the newly kept boxes are appended to the kept list (shared memory, spilling to the output rows in global).
// Work ~ N x kept IoUs instead of N^2, and the sequential part is proportional to the number of kept boxes.
// IoU arithmetic is torchvision's CUDA devIoU, same-class pairs only (class-aware variant); see nms_hit for its rounding.
constexpr int kNmsChunk = 256;
constexpr int kNmsKeepSmem = 3072;

// IoU(a, b) > thr of an earlier box a (higher in the score order) and a later box b, rounded as torchvision's CUDA devIoU is
// compiled: widths, heights, the intersection and a's area are rounded products, b's area is fused into the union
// (union = fmaf(wb, hb, area_a) - inter), an IEEE divide and a float compare.  The _rn intrinsics pin that order: with plain
// operators nvcc picks which area it fuses (per call site, after hoisting), and a one-ulp difference in the union flips pairs
// within an ulp of the threshold.
__device__ __forceinline__ bool nms_hit(const float4 a, const float4 b, float thr) {
  const float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y);
  const float xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
  const float w = fmaxf(__fsub_rn(xx2, xx1), 0.f), h = fmaxf(__fsub_rn(yy2, yy1), 0.f);
  const float inter = __fmul_rn(w, h);
  const float sa = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  const float uni = __fsub_rn(__fmaf_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y), sa), inter);
  return __fdiv_rn(inter, uni) > thr;
}

// kAgnostic: every pair is tested, whatever the classes (torchvision.ops.nms of postprocess(..., class_agnostic=True)).
template <bool kAgnostic>
__global__ void __launch_bounds__(1024) nms_greedy_kernel(PostSlices sl, float thr, float* __restrict__ out, int* __restrict__ out_count,
                                                           int max_keep, int* __restrict__ out_anchor) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int img = blockIdx.x;
  const float* const sorted = sl.sorted(img);
  const int* const count = sl.count(img);
  const int* const sorted_anchor = sl.sorted_anchor(img);
  out += static_cast<long>(img) * sl.A * 7;
  out_count += img;
  if (out_anchor) out_anchor += static_cast<long>(img) * sl.A;
  extern __shared__ float4 kept_box[];                       // [kNmsKeepSmem]
  float* kept_cls = reinterpret_cast<float*>(kept_box + kNmsKeepSmem);  // [kNmsKeepSmem]
  __shared__ float4 cbox[kNmsChunk];
  __shared__ float ccls[kNmsChunk];
  __shared__ unsigned long long pair_mask[kNmsChunk][4];
  __shared__ unsigned long long alive_w[4], kept_w[4];
  __shared__ int nk_s;
  const int n = *count;
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) nk_s = 0;
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += kNmsChunk) {
    const int nk = nk_s;
    if (nk >= max_keep) break;  // uniform: the first max_keep rows of the full result are already final
    const int ci = tid >> 2, sub = tid & 3;  // candidate within chunk, quarter of the kept list
    const int j = c0 + ci;
    float4 bx = make_float4(0.f, 0.f, 0.f, 0.f);
    float cl = -1.f;
    if (j < n) {
      const float* d = sorted + static_cast<long>(j) * 7;
      bx = make_float4(d[0], d[1], d[2], d[3]);
      cl = d[6];
    }
    bool sup = (j >= n);
    for (int k = sub; k < nk && !sup; k += 4) {
      float4 kb;
      float kc;
      if (k < kNmsKeepSmem) { kb = kept_box[k]; kc = kept_cls[k]; }
      else { const float* d = out + static_cast<long>(k) * 7; kb = make_float4(d[0], d[1], d[2], d[3]); kc = d[6]; }
      if ((kAgnostic || kc == cl) && nms_hit(kb, bx, thr)) sup = true;
    }
    sup |= __shfl_xor_sync(0xffffffffu, sup, 1) != 0;
    sup |= __shfl_xor_sync(0xffffffffu, sup, 2) != 0;
    if (sub == 0) { cbox[ci] = bx; ccls[ci] = cl; }
    // alive words: ballot over lanes with sub == 0 (8 candidates per warp)
    const unsigned bal = __ballot_sync(0xffffffffu, !sup && sub == 0);
    if (tid < 4) alive_w[tid] = 0ull;
    __syncthreads();
    if (lane == 0) {
      // compress ballot bits (every 4th lane) into 8 bits at position (warp*8)
      unsigned v = 0;
      for (int t = 0; t < 8; ++t) v |= ((bal >> (4 * t)) & 1u) << t;
      const int cbase = (tid >> 5) * 8;  // first candidate of this warp
      atomicOr(&alive_w[cbase >> 6], static_cast<unsigned long long>(v) << (cbase & 63));
    }
    __syncthreads();
    {  // pairwise bits inside the chunk: candidate ci vs candidates [sub*64, sub*64+64), later ones only
      unsigned long long bits = 0ull;
      const bool me = (alive_w[ci >> 6] >> (ci & 63)) & 1ull;
      if (me) {
        const unsigned long long aw = alive_w[sub];
        for (int t = 0; t < 64; ++t) {
          const int o = sub * 64 + t;
          if (o > ci && ((aw >> t) & 1ull) && (kAgnostic || ccls[o] == cl) && nms_hit(bx, cbox[o], thr)) bits |= 1ull << t;
        }
      }
      pair_mask[ci][sub] = bits;
    }
    __syncthreads();
    if (tid < 32) {  // greedy resolution of the chunk (all lanes run the same scalar code)
      unsigned long long removed[4] = {0ull, 0ull, 0ull, 0ull};
      unsigned long long kept[4] = {0ull, 0ull, 0ull, 0ull};
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        unsigned long long cur = ~alive_w[w] | removed[w];
        while (~cur != 0ull) {
          const int t = __ffsll(static_cast<long long>(~cur)) - 1;
          kept[w] |= 1ull << t;
          const int r = w * 64 + t;
          cur |= pair_mask[r][w] | (1ull << t);
#pragma unroll
          for (int w2 = w + 1; w2 < 4; ++w2) removed[w2] |= pair_mask[r][w2];
        }
      }
      if (tid == 0) { kept_w[0] = kept[0]; kept_w[1] = kept[1]; kept_w[2] = kept[2]; kept_w[3] = kept[3]; }
    }
    __syncthreads();
    if (tid < kNmsChunk) {
      const int w = tid >> 6, t = tid & 63;
      if ((kept_w[w] >> t) & 1ull) {
        int pos = nk + __popcll(kept_w[w] & ((1ull << t) - 1ull));
        for (int w2 = 0; w2 < w; ++w2) pos += __popcll(kept_w[w2]);
        if (pos < kNmsKeepSmem) { kept_box[pos] = cbox[tid]; kept_cls[pos] = ccls[tid]; }
        const float* d = sorted + static_cast<long>(c0 + tid) * 7;
        float* o = out + static_cast<long>(pos) * 7;
#pragma unroll
        for (int q = 0; q < 7; ++q) o[q] = d[q];
        if (out_anchor) out_anchor[pos] = sorted_anchor[c0 + tid];
      }
    }
    __syncthreads();
    if (tid == 0) nk_s = nk + __popcll(kept_w[0]) + __popcll(kept_w[1]) + __popcll(kept_w[2]) + __popcll(kept_w[3]);
    __syncthreads();
  }
  if (tid == 0) *out_count = min(nk_s, max_keep);
}

}  // namespace uc

using namespace uc;

static int make_levels(const char* what, const float* const* regobj, const float* const* cls, const int* hw, const int* strides, int ld_ro,
                       int ld_cls, const long* bs_ro, const long* bs_cls, int ncls, int B, DecodeLevels& lv) {
  if (!regobj || !cls || !hw || !strides || ncls < 1 || ncls > ld_cls || ld_ro < 5) return set_error(UC_EINVAL, "%s: bad arguments", what);
  if (B < 1) return set_error(UC_EINVAL, "%s: B must be >= 1 (got %d)", what, B);
  int start = 0;
  for (int k = 0; k < 3; ++k) {
    lv.regobj[k] = regobj[k]; lv.cls[k] = cls[k];
    lv.h[k] = hw[2 * k]; lv.w[k] = hw[2 * k + 1]; lv.stride[k] = strides[k]; lv.start[k] = start;
    const long hwk = static_cast<long>(lv.h[k]) * lv.w[k];
    lv.bs_ro[k] = B > 1 ? bs_ro[k] : hwk * ld_ro;
    lv.bs_cls[k] = B > 1 ? bs_cls[k] : hwk * ld_cls;
    if (lv.bs_ro[k] < hwk * ld_ro || lv.bs_cls[k] < hwk * ld_cls)
      return set_error(UC_EINVAL, "%s: bad per-image strides of level %d (need >= h*w*ld)", what, k);
    start += lv.h[k] * lv.w[k];
  }
  lv.ld_ro = ld_ro; lv.ld_cls = ld_cls; lv.ncls = ncls; lv.total = start;
  return UC_OK;
}

static int head_decode(const char* what, const float* const* regobj, const float* const* cls, const int* hw, const int* strides, int ld_ro,
                       int ld_cls, const long* bs_ro, const long* bs_cls, int ncls, int B, float* out, void* stream_v) {
  if (!out) return set_error(UC_EINVAL, "%s: bad arguments", what);
  DecodeLevels lv;
  if (int e = make_levels(what, regobj, cls, hw, strides, ld_ro, ld_cls, bs_ro, bs_cls, ncls, B, lv)) return e;
  launch_pdl(head_decode_kernel, dim3((lv.total + 255) / 256, B), 256, 0, static_cast<cudaStream_t>(stream_v), lv, out);
  return check_launch(what);
}

extern "C" int uc_head_decode(const float* const* regobj, const float* const* cls, const int* hw, const int* strides, int ld_ro,
                              int ld_cls, int ncls, float* out, void* stream_v) {
  return head_decode("uc_head_decode", regobj, cls, hw, strides, ld_ro, ld_cls, nullptr, nullptr, ncls, 1, out, stream_v);
}

extern "C" int uc_head_decode_batched(const float* const* regobj, const float* const* cls, const int* hw, const int* strides, int ld_ro,
                                      int ld_cls, const long* bs_ro, const long* bs_cls, int ncls, int B, float* out, void* stream_v) {
  if (B > 1 && (!bs_ro || !bs_cls)) return set_error(UC_EINVAL, "uc_head_decode_batched: null per-image strides");
  return head_decode("uc_head_decode_batched", regobj, cls, hw, strides, ld_ro, ld_cls, bs_ro, bs_cls, ncls, B, out, stream_v);
}

extern "C" long uc_postprocess_workspace_bytes(int max_anchors) {
  const long A = max_anchors;
  long a2 = 1;
  while (a2 < A) a2 <<= 1;
  return A * 7 * 4 * 2 + a2 * 8 + A * 4 * 2 + 256;
}

extern "C" long uc_postprocess_workspace_bytes_batched(int max_anchors, int B) {
  return B < 1 ? 0 : B * uc_postprocess_workspace_bytes(max_anchors);
}

static PostSlices make_slices(void* workspace, int A) {
  long a2 = 1;
  while (a2 < A) a2 <<= 1;
  PostSlices sl;
  sl.ws = static_cast<uint8_t*>(workspace);
  sl.per_image = uc_postprocess_workspace_bytes(A);
  sl.a2 = a2;
  sl.A = A;
  return sl;
}

static int check_workspace(const char* what, int A, int B, long workspace_bytes) {
  if (B < 1) return set_error(UC_EINVAL, "%s: B must be >= 1 (got %d)", what, B);
  if (workspace_bytes < B * uc_postprocess_workspace_bytes(A))
    return set_error(UC_EINVAL, "%s: workspace too small (%ld bytes for %d images of %d anchors, need %ld)", what, workspace_bytes, B, A,
                     B * uc_postprocess_workspace_bytes(A));
  return UC_OK;
}

template <bool kAgnostic>
static void launch_nms(const PostSlices& sl, int B, float nms_thre, float* out_dets, int* out_count, int max_keep, int* out_anchor,
                       cudaStream_t stream) {
  constexpr int smem = kNmsKeepSmem * (16 + 4);
  static PerDeviceFlag attr_dev;
  bool& attr = attr_dev.get();
  if (!attr) {
    cudaFuncSetAttribute(nms_greedy_kernel<kAgnostic>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = true;
  }
  launch_pdl(nms_greedy_kernel<kAgnostic>, B, 1024, smem, stream, sl, nms_thre, out_dets, out_count, max_keep > 0 ? max_keep : 0x7fffffff,
             out_anchor);
}

// sort, gather and greedy NMS of the candidates a filter left in the workspace
static void launch_nms_stages(const PostSlices& sl, int B, float nms_thre, int max_keep, int flags, float* out_dets, int* out_count,
                              int* out_anchor, cudaStream_t stream) {
  launch_pdl(sort_desc_kernel, B, 1024, 0, stream, sl);
  launch_pdl(det_gather_kernel, dim3(std::min(num_sms() * 4, (sl.A + 255) / 256), B), 256, 0, stream, sl);
  if (flags & UC_POST_CLASS_AGNOSTIC)
    launch_nms<true>(sl, B, nms_thre, out_dets, out_count, max_keep, out_anchor, stream);
  else
    launch_nms<false>(sl, B, nms_thre, out_dets, out_count, max_keep, out_anchor, stream);
}

static int postprocess(const char* what, const float* pred, int A, int ncls, float conf_thre, float nms_thre, int max_keep, int B, int flags,
                       void* workspace, long workspace_bytes, float* out_dets, int* out_count, int* out_anchor, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!pred || !workspace || !out_dets || !out_count || A < 1 || ncls < 1) return set_error(UC_EINVAL, "%s: bad arguments", what);
  if (flags & ~UC_POST_CLASS_AGNOSTIC) return set_error(UC_EINVAL, "%s: unknown flags 0x%x", what, flags);
  if (int e = check_workspace(what, A, B, workspace_bytes)) return e;
  const PostSlices sl = make_slices(workspace, A);
  launch_pdl(det_filter_kernel, B, 1024, 0, stream, pred, A, ncls, conf_thre, sl);
  launch_nms_stages(sl, B, nms_thre, max_keep, flags, out_dets, out_count, out_anchor, stream);
  return check_launch(what);
}

extern "C" int uc_postprocess(const float* pred, int A, int ncls, float conf_thre, float nms_thre, int max_keep, void* workspace,
                              long workspace_bytes, float* out_dets, int* out_count, int* out_anchor, void* stream_v) {
  return postprocess("uc_postprocess", pred, A, ncls, conf_thre, nms_thre, max_keep, 1, 0, workspace, workspace_bytes, out_dets, out_count,
                     out_anchor, stream_v);
}

extern "C" int uc_postprocess_batched(const float* pred, int A, int ncls, float conf_thre, float nms_thre, int max_keep, int B,
                                      void* workspace, long workspace_bytes, float* out_dets, int* out_count, int* out_anchor,
                                      void* stream_v) {
  return postprocess("uc_postprocess_batched", pred, A, ncls, conf_thre, nms_thre, max_keep, B, 0, workspace, workspace_bytes, out_dets,
                     out_count, out_anchor, stream_v);
}

extern "C" int uc_postprocess_batched_ex(const float* pred, int A, int ncls, float conf_thre, float nms_thre, int max_keep, int B, int flags,
                                         void* workspace, long workspace_bytes, float* out_dets, int* out_count, int* out_anchor,
                                         void* stream_v) {
  return postprocess("uc_postprocess_batched_ex", pred, A, ncls, conf_thre, nms_thre, max_keep, B, flags, workspace, workspace_bytes,
                     out_dets, out_count, out_anchor, stream_v);
}

extern "C" int uc_det_candidates_batched(const float* const* regobj, const float* const* cls, const int* hw, const int* strides, int ld_ro,
                                         int ld_cls, const long* bs_ro, const long* bs_cls, int ncls, int B, float conf_thre,
                                         void* workspace, long workspace_bytes, void* stream_v) {
  const char* what = "uc_det_candidates_batched";
  if (!workspace) return set_error(UC_EINVAL, "%s: null workspace", what);
  if (B > 1 && (!bs_ro || !bs_cls)) return set_error(UC_EINVAL, "%s: null per-image strides", what);
  DecodeLevels lv;
  if (int e = make_levels(what, regobj, cls, hw, strides, ld_ro, ld_cls, bs_ro, bs_cls, ncls, B, lv)) return e;
  if (int e = check_workspace(what, lv.total, B, workspace_bytes)) return e;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const PostSlices sl = make_slices(workspace, lv.total);
  const int tile = cand_tile(lv.total), ntiles = (lv.total + tile - 1) / tile;
  launch_pdl(det_candidates_kernel, dim3(ntiles, B), kCandThreads, 0, stream, lv, tile, conf_thre, sl);
  launch_pdl(det_candidates_compact_kernel, dim3(ntiles, B), kCandThreads, 0, stream, tile, sl);
  return check_launch(what);
}

extern "C" int uc_postprocess_nms_batched(int A, float nms_thre, int max_keep, int B, int flags, void* workspace, long workspace_bytes,
                                          float* out_dets, int* out_count, int* out_anchor, void* stream_v) {
  const char* what = "uc_postprocess_nms_batched";
  if (!workspace || !out_dets || !out_count || A < 1) return set_error(UC_EINVAL, "%s: bad arguments", what);
  if (flags & ~UC_POST_CLASS_AGNOSTIC) return set_error(UC_EINVAL, "%s: unknown flags 0x%x", what, flags);
  if (int e = check_workspace(what, A, B, workspace_bytes)) return e;
  launch_nms_stages(make_slices(workspace, A), B, nms_thre, max_keep, flags, out_dets, out_count, out_anchor,
                    static_cast<cudaStream_t>(stream_v));
  return check_launch(what);
}
