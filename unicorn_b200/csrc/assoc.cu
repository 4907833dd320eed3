// Instance-embedding sampling and association scoring for the MOT path.
//   uc_sample_embed   unicorn/evaluators/mot_evaluator.py:1024-1034 (one F.grid_sample per box in the reference); the
//                     _batched entry point samples B images (B sequences' frames) in one launch
//   uc_bisoftmax      unicorn/tracker/quasi_dense_embed_tracker.py:166-175 (feats = E M^T, bi-softmax, class gate)
//   uc_box_iou        torchvision.ops.box_iou as used at quasi_dense_embed_tracker.py:80,146
// All three are tiny (N, M <= a few hundred): one launch each, fp32 arithmetic in the reference's operation order.
#include "uc_common.h"
#include "../../include/unicorn_b200.h"

namespace uc {

// one warp per box, lane owns channels lane, lane+32, ...  embed NHWC 16-bit [h,w,C]; blockIdx.y = image: image b reads
// embed + b * bs_embed, boxes + b * bs_boxes and count[b], and writes out + b * bs_out
__global__ void __launch_bounds__(256) sample_embed_kernel(const uint16_t* __restrict__ embed, int ld, long bs_embed, int h, int w, int C,
                                                            int dtype, const float* __restrict__ boxes, int ldb, long bs_boxes,
                                                            const int* __restrict__ count, int n_max, float stride, float* __restrict__ out,
                                                            long bs_out) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int b = blockIdx.y;
  const int n = count ? min(count[b], n_max) : n_max;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  embed += b * bs_embed;
  out += b * bs_out;
  const float* bx = boxes + b * bs_boxes + static_cast<long>(i) * ldb;
  // centre in embedding-map pixels, clamped, normalised to [-1,1] exactly as the reference does ...
  float cx = (bx[0] + bx[2]) / 2 / stride - 0.5f, cy = (bx[1] + bx[3]) / 2 / stride - 0.5f;
  cx = (fminf(fmaxf(cx, 0.f), static_cast<float>(w - 1)) / (w - 1) - 0.5f) * 2.0f;
  cy = (fminf(fmaxf(cy, 0.f), static_cast<float>(h - 1)) / (h - 1) - 0.5f) * 2.0f;
  // ... then grid_sample(bilinear, padding_mode=border, align_corners=False): unnormalise, clip to the border
  float x = ((cx + 1.f) * w - 1.f) / 2.f, y = ((cy + 1.f) * h - 1.f) / 2.f;
  x = fminf(fmaxf(x, 0.f), static_cast<float>(w - 1));
  y = fminf(fmaxf(y, 0.f), static_cast<float>(h - 1));
  const int x0 = static_cast<int>(floorf(x)), y0 = static_cast<int>(floorf(y));
  const int x1 = min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1);
  const float lx = x - x0, ly = y - y0;
  const float w00 = (1.f - lx) * (1.f - ly), w01 = lx * (1.f - ly), w10 = (1.f - lx) * ly, w11 = lx * ly;
  for (int c = lane; c < C; c += 32) {
    const float v00 = bits16_to_float(embed[(static_cast<long>(y0) * w + x0) * ld + c], dtype);
    const float v01 = bits16_to_float(embed[(static_cast<long>(y0) * w + x1) * ld + c], dtype);
    const float v10 = bits16_to_float(embed[(static_cast<long>(y1) * w + x0) * ld + c], dtype);
    const float v11 = bits16_to_float(embed[(static_cast<long>(y1) * w + x1) * ld + c], dtype);
    out[static_cast<long>(i) * C + c] = v00 * w00 + v01 * w01 + v10 * w10 + v11 * w11;
  }
}

// feats[i,j] = <E_i, M_j>; one block computes the whole matrix into global, then row / column softmax passes.
__global__ void __launch_bounds__(256) feats_kernel(const float* __restrict__ E, const float* __restrict__ Mm, int N, int M, int C,
                                                     float* __restrict__ feats) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const int i = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || j >= M) return;
  float acc = 0.f;
  for (int c = 0; c < C; ++c) acc = fmaf(E[static_cast<long>(i) * C + c], Mm[static_cast<long>(j) * C + c], acc);
  feats[static_cast<long>(i) * M + j] = acc;
}
__global__ void __launch_bounds__(128) softmax_stats_kernel(const float* __restrict__ feats, int N, int M, float* __restrict__ rmax,
                                                            float* __restrict__ rsum, float* __restrict__ cmax, float* __restrict__ csum) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  // blocks [0,N): row i ; blocks [N, N+M): column j
  __shared__ float red[128];
  const bool is_row = blockIdx.x < N;
  const int idx = is_row ? blockIdx.x : blockIdx.x - N;
  const int len = is_row ? M : N;
  const long s0 = is_row ? static_cast<long>(idx) * M : idx, st = is_row ? 1 : M;
  float mx = -INFINITY;
  for (int t = threadIdx.x; t < len; t += 128) mx = fmaxf(mx, feats[s0 + t * st]);
  red[threadIdx.x] = mx;
  __syncthreads();
  for (int o = 64; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + o]); __syncthreads(); }
  mx = red[0];
  __syncthreads();
  float sm = 0.f;
  for (int t = threadIdx.x; t < len; t += 128) sm += expf(feats[s0 + t * st] - mx);
  red[threadIdx.x] = sm;
  __syncthreads();
  for (int o = 64; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) { (is_row ? rmax : cmax)[idx] = mx; (is_row ? rsum : csum)[idx] = red[0]; }
}
__global__ void __launch_bounds__(256) bisoftmax_kernel(const float* __restrict__ feats, int N, int M, const float* __restrict__ rmax,
                                                         const float* __restrict__ rsum, const float* __restrict__ cmax,
                                                         const float* __restrict__ csum, const float* __restrict__ lab_d,
                                                         const float* __restrict__ lab_m, float* __restrict__ scores) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const long t = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<long>(N) * M) return;
  const int i = static_cast<int>(t / M), j = static_cast<int>(t % M);
  const float f = feats[t];
  float s = (expf(f - rmax[i]) / rsum[i] + expf(f - cmax[j]) / csum[j]) / 2;
  if (lab_d && lab_m && lab_d[i] != lab_m[j]) s = 0.f;
  scores[t] = s;
}

// plus1 = 0: torchvision.ops.box_iou; plus1 = 1: cython_bbox.bbox_overlaps (inclusive-pixel convention used by ByteTrack,
// unicorn/tracker/matching.py:65-68).  Every step is rounded on its own, as torchvision's separate torch ops are
// (union = rn(rn(area1 + area2) - inter)): the _rn intrinsics keep nvcc from fusing an area's product into the union, so
// plus1 = 0 equals torchvision.ops.box_iou bit for bit.  plus1 = 1 is the same order with the + 1 after each difference;
// bbox_overlaps computes in float64.
__global__ void __launch_bounds__(256) box_iou_kernel(const float* __restrict__ a, int lda, int N, const float* __restrict__ b, int ldb,
                                                       int M, float* __restrict__ out, float plus1) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const long t = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<long>(N) * M) return;
  const float* p = a + (t / M) * lda;
  const float* q = b + (t % M) * ldb;
  const float area1 = __fmul_rn(__fadd_rn(__fsub_rn(p[2], p[0]), plus1), __fadd_rn(__fsub_rn(p[3], p[1]), plus1));
  const float area2 = __fmul_rn(__fadd_rn(__fsub_rn(q[2], q[0]), plus1), __fadd_rn(__fsub_rn(q[3], q[1]), plus1));
  const float w = fmaxf(__fadd_rn(__fsub_rn(fminf(p[2], q[2]), fmaxf(p[0], q[0])), plus1), 0.f);
  const float h = fmaxf(__fadd_rn(__fsub_rn(fminf(p[3], q[3]), fmaxf(p[1], q[1])), plus1), 0.f);
  const float inter = __fmul_rn(w, h);
  out[t] = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area1, area2), inter));
}


// Greedy assignment of the quasi-dense tracker (unicorn/tracker/quasi_dense_embed_tracker.py:188-199): detections in descending
// score order; row i takes its best memo column j (first maximum, like torch.max) if conf > match_thr and the column is a tracklet
// (memo id > -1): with det score > obj_thr it gets the id and the column is zeroed for every other row, otherwise conf > nms_conf_thr
// marks it -2.  Inherently sequential over rows (N <= a few hundred): one CTA, the column search is parallel.
__global__ void __launch_bounds__(256) qd_assign_kernel(const float* __restrict__ scores, int N, int M, const long long* __restrict__ memo_ids,
                                                         const float* __restrict__ det_scores, int lds, float match_thr, float obj_thr,
                                                         float nms_conf_thr, long long* __restrict__ ids, uint8_t* __restrict__ taken) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float s_val[256];
  __shared__ int s_idx[256];
  for (int j = threadIdx.x; j < M; j += blockDim.x) taken[j] = 0;
  __syncthreads();
  for (int i = 0; i < N; ++i) {
    float best = -1.f;  // scores are >= 0
    int bj = 0x7fffffff;
    for (int j = threadIdx.x; j < M; j += blockDim.x) {
      const float v = taken[j] ? 0.f : scores[static_cast<long>(i) * M + j];
      if (v > best) { best = v; bj = j; }  // strict: the earliest index of this thread's stride wins ties
    }
    s_val[threadIdx.x] = best;
    s_idx[threadIdx.x] = bj;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
      if (threadIdx.x < o) {
        const float v = s_val[threadIdx.x + o];
        const int jj = s_idx[threadIdx.x + o];
        if (v > s_val[threadIdx.x] || (v == s_val[threadIdx.x] && jj < s_idx[threadIdx.x])) { s_val[threadIdx.x] = v; s_idx[threadIdx.x] = jj; }
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      const float conf = s_val[0];
      const int j = s_idx[0];
      long long id = -1;
      if (M > 0 && conf > match_thr && memo_ids[j] > -1) {
        if (det_scores[static_cast<long>(i) * lds] > obj_thr) { id = memo_ids[j]; taken[j] = 1; }
        else if (conf > nms_conf_thr) id = -2;
      }
      ids[i] = id;
    }
    __syncthreads();
  }
}

}  // namespace uc

using namespace uc;

static int sample_embed(const char* name, const void* embed, int ld, long bs_embed, int h, int w, int C, int dtype, const float* boxes,
                        int ldb, long bs_boxes, const int* count_dev, int n_max, float stride, float* out, long bs_out, int B,
                        cudaStream_t stream) {
  if (n_max == 0) return UC_OK;
  launch_pdl(sample_embed_kernel, dim3((n_max + 7) / 8, B), 256, 0, stream, static_cast<const uint16_t*>(embed), ld, bs_embed, h, w, C, dtype,
             boxes, ldb, bs_boxes, count_dev, n_max, stride, out, bs_out);
  return check_launch(name);
}

extern "C" int uc_sample_embed(const void* embed, int ld, int h, int w, int C, int dtype, const float* boxes, int ldb,
                               const int* count_dev, int n_max, float stride, float* out, void* stream_v) {
  if (!embed || !boxes || !out || n_max < 0 || h < 2 || w < 2 || ldb < 4) return set_error(UC_EINVAL, "uc_sample_embed: bad arguments");
  return sample_embed("uc_sample_embed", embed, ld, 0, h, w, C, dtype, boxes, ldb, 0, count_dev, n_max, stride, out, 0, 1,
                      static_cast<cudaStream_t>(stream_v));
}

extern "C" int uc_sample_embed_batched(const void* embed, int ld, long bs_embed, int h, int w, int C, int dtype, const float* boxes, int ldb,
                                       long bs_boxes, const int* count_dev, int n_max, float stride, float* out, long bs_out, int B,
                                       void* stream_v) {
  if (B < 1) return set_error(UC_EINVAL, "uc_sample_embed_batched: B must be >= 1");
  if (!embed || !boxes || !count_dev || !out) return set_error(UC_EINVAL, "uc_sample_embed_batched: null pointer");
  if (n_max < 0 || h < 2 || w < 2 || C < 1 || ld < C || ldb < 4) return set_error(UC_EINVAL, "uc_sample_embed_batched: bad arguments");
  if (bs_embed < static_cast<long>(h) * w * ld || bs_boxes < static_cast<long>(n_max) * ldb || bs_out < static_cast<long>(n_max) * C)
    return set_error(UC_EINVAL, "uc_sample_embed_batched: bad per-image strides (each must cover one image)");
  return sample_embed("uc_sample_embed_batched", embed, ld, bs_embed, h, w, C, dtype, boxes, ldb, bs_boxes, count_dev, n_max, stride, out,
                      bs_out, B, static_cast<cudaStream_t>(stream_v));
}

extern "C" int uc_bisoftmax(const float* det_embeds, const float* memo_embeds, int N, int M, int C, const float* det_labels,
                            const float* memo_labels, float* workspace, float* scores, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!det_embeds || !memo_embeds || !workspace || !scores || N < 1 || M < 1) return set_error(UC_EINVAL, "uc_bisoftmax: bad arguments");
  float* feats = workspace;  // [N*M] + 2N + 2M floats
  float* rmax = feats + static_cast<long>(N) * M;
  float* rsum = rmax + N;
  float* cmax = rsum + N;
  float* csum = cmax + M;
  launch_pdl(feats_kernel, dim3((M + 255) / 256, N), 256, 0, stream, det_embeds, memo_embeds, N, M, C, feats);
  launch_pdl(softmax_stats_kernel, N + M, 128, 0, stream, feats, N, M, rmax, rsum, cmax, csum);
  launch_pdl(bisoftmax_kernel, static_cast<unsigned>((static_cast<long>(N) * M + 255) / 256), 256, 0, stream, feats, N, M, rmax, rsum, cmax, csum,
                                                                                                     det_labels, memo_labels, scores);
  return check_launch("uc_bisoftmax");
}

extern "C" int uc_box_iou(const float* a, int lda, int N, const float* b, int ldb, int M, float* out, int plus_one, void* stream_v) {
  if (!a || !b || !out || N < 1 || M < 1 || lda < 4 || ldb < 4) return set_error(UC_EINVAL, "uc_box_iou: bad arguments");
  launch_pdl(box_iou_kernel, static_cast<unsigned>((static_cast<long>(N) * M + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_v), a, lda, N, b, ldb, M, out, plus_one ? 1.f : 0.f);
  return check_launch("uc_box_iou");
}

extern "C" int uc_qd_assign(const float* scores, int N, int M, const long long* memo_ids, const float* det_scores, int ld_det, float match_thr,
                            float obj_thr, float nms_conf_thr, long long* ids_out, uint8_t* taken_ws, void* stream_v) {
  if (N < 0 || M < 0 || (N > 0 && (!det_scores || !ids_out)) || (N > 0 && M > 0 && (!scores || !memo_ids || !taken_ws)))
    return set_error(UC_EINVAL, "uc_qd_assign: bad arguments");
  if (N == 0) return UC_OK;
  launch_pdl(qd_assign_kernel, 1, 256, 0, static_cast<cudaStream_t>(stream_v), scores, N, M, memo_ids, det_scores, ld_det, match_thr, obj_thr,
             nms_conf_thr, ids_out, taken_ws);
  return check_launch("uc_qd_assign");
}
