// Multi-scale deformable attention sampling (forward only).
//  * uc_msda_forward_f32  — drop-in for the reference operator MultiScaleDeformableAttention.ms_deform_attn_forward
//    (unicorn/models/ops/src/ms_deform_attn.h:20-39 -> cuda/ms_deform_attn_cuda.cu:20-80 ->
//     ms_deformable_im2col_gpu_kernel, cuda/ms_deform_im2col_cuda.cuh:237-299, bilinear :33-84).
//  * uc_msda_fused_bf16   — the form the H100 path uses: reads the raw sampling-offset / attention-logit projection
//    (one fused Linear), does the softmax over L*P, the reference-point arithmetic
//    (deformable_transformer.py:141-153, ops/modules/ms_deform_attn.py:99-105) and the gather in one kernel.
// Semantics (both): pixel coords x = loc_x*W - 0.5, y = loc_y*H - 0.5; a sample counts only if -1 < y < H and
// -1 < x < W; out-of-map corners contribute zero.  The gather is L2-resident (value is 4 MB at 800x1280).
#include "uc_common.h"
#include "../../include/unicorn_b200.h"
#include <algorithm>

namespace uc {

__global__ void __launch_bounds__(256) msda_f32_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                                                        const int64_t* __restrict__ lstart, const float* __restrict__ loc,
                                                        const float* __restrict__ attn, float* __restrict__ out, int B, int S,
                                                        int M, int D, int L, int Lq, int P) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const long total = static_cast<long>(B) * Lq * M * D;
  for (long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(i % D);
    long t = i / D;
    const int m = static_cast<int>(t % M);
    t /= M;
    const int q = static_cast<int>(t % Lq);
    const int b = static_cast<int>(t / Lq);
    const float* lp = loc + ((static_cast<long>(b) * Lq + q) * M + m) * L * P * 2;
    const float* ap = attn + ((static_cast<long>(b) * Lq + q) * M + m) * L * P;
    float acc = 0.f;
    for (int l = 0; l < L; ++l) {
      const int H = static_cast<int>(shapes[2 * l]), W = static_cast<int>(shapes[2 * l + 1]);
      const float* vb = value + (static_cast<long>(b) * S + lstart[l]) * M * D + m * D + d;
      for (int p = 0; p < P; ++p) {
        const float lx = lp[(l * P + p) * 2], ly = lp[(l * P + p) * 2 + 1];
        const float a = ap[l * P + p];
        const float h_im = ly * H - 0.5f, w_im = lx * W - 0.5f;
        if (h_im > -1.f && w_im > -1.f && h_im < H && w_im < W) {
          const int h0 = static_cast<int>(floorf(h_im)), w0 = static_cast<int>(floorf(w_im));
          const float lh = h_im - h0, lw = w_im - w0, hh = 1.f - lh, hw = 1.f - lw;
          const long rs = static_cast<long>(M) * D;
          float v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f;
          if (h0 >= 0 && w0 >= 0) v1 = vb[(static_cast<long>(h0) * W + w0) * rs];
          if (h0 >= 0 && w0 + 1 <= W - 1) v2 = vb[(static_cast<long>(h0) * W + w0 + 1) * rs];
          if (h0 + 1 <= H - 1 && w0 >= 0) v3 = vb[(static_cast<long>(h0 + 1) * W + w0) * rs];
          if (h0 + 1 <= H - 1 && w0 + 1 <= W - 1) v4 = vb[(static_cast<long>(h0 + 1) * W + w0 + 1) * rs];
          acc += a * (hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4);
        }
      }
    }
    out[i] = acc;
  }
}

struct MsdaLevels {
  int H[4], W[4], start[4];
};

// 8 lanes per (image, query, head); each lane owns 4 of the head's 32 channels.  Rows (value, offlog, out) are level-major,
// images within a level: level l of image b starts at row B * start[l] + b * H[l] * W[l] (for B = 1 the concatenation of the
// levels).  value bf16 rows of M*32; offlog fp32 rows of M*L*P*2 + M*L*P; an image's queries are its levels' pixel grids (query
// qi of level ql at pixel (qy,qx)), and the reference point (qx+0.5)/Wq, (qy+0.5)/Hq is shared by all levels of that image.
__global__ void __launch_bounds__(256) msda_fused_kernel(const uint2* __restrict__ value, const float* __restrict__ offlog,
                                                          uint2* __restrict__ out, MsdaLevels lv, int M, int L, int P, int Lq,
                                                          int ld_offlog, int B) {
  pdl_wait();               // programmatic dependent launch: global memory is touched only after the predecessor completed
  pdl_launch_dependents();  // ... and the next kernel in the stream may become resident / run its prologue from here on
  const long g = (static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 3;  // (b, q, m)
  const int sub = threadIdx.x & 7;
  if (g >= static_cast<long>(B) * Lq * M) return;
  const int b = static_cast<int>(g / (static_cast<long>(Lq) * M));
  const int qm = static_cast<int>(g - static_cast<long>(b) * Lq * M);
  const int qq = qm / M, m = qm % M;
  int ql = 0;
  while (ql + 1 < L && qq >= lv.start[ql + 1]) ++ql;
  const int qi = qq - lv.start[ql];
  const long q = static_cast<long>(B) * lv.start[ql] + static_cast<long>(b) * lv.H[ql] * lv.W[ql] + qi;  // row of this query
  const float rx = ((qi % lv.W[ql]) + 0.5f) / lv.W[ql], ry = ((qi / lv.W[ql]) + 0.5f) / lv.H[ql];
  const int LP = L * P;
  const float* off = offlog + q * ld_offlog + m * LP * 2;
  const float* lg = offlog + q * ld_offlog + M * LP * 2 + m * LP;
  float mx = -INFINITY;
  for (int i = 0; i < LP; ++i) mx = fmaxf(mx, __ldg(lg + i));
  float den = 0.f;
  for (int i = 0; i < LP; ++i) den += __expf(__ldg(lg + i) - mx);
  const float inv = 1.f / den;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const int rs = M * 8;  // row stride in uint2 (4 bf16)
  for (int l = 0; l < L; ++l) {
    const int H = lv.H[l], W = lv.W[l];
    const uint2* vb = value + (static_cast<long>(B) * lv.start[l] + static_cast<long>(b) * H * W) * rs + m * 8 + sub;
    for (int p = 0; p < P; ++p) {
      const float a = __expf(__ldg(lg + l * P + p) - mx) * inv;
      const float lx = rx + __ldg(off + (l * P + p) * 2) / W, ly = ry + __ldg(off + (l * P + p) * 2 + 1) / H;
      const float h_im = ly * H - 0.5f, w_im = lx * W - 0.5f;
      if (h_im > -1.f && w_im > -1.f && h_im < H && w_im < W) {
        const int h0 = static_cast<int>(floorf(h_im)), w0 = static_cast<int>(floorf(w_im));
        const float lh = h_im - h0, lw = w_im - w0, hh = 1.f - lh, hw = 1.f - lw;
        const float cw[4] = {hh * hw * a, hh * lw * a, lh * hw * a, lh * lw * a};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int yy = h0 + (c >> 1), xx = w0 + (c & 1);
          if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
            const uint2 u = __ldg(vb + (static_cast<long>(yy) * W + xx) * rs);
            acc[0] = fmaf(cw[c], bf16lo(u.x), acc[0]); acc[1] = fmaf(cw[c], bf16hi(u.x), acc[1]);
            acc[2] = fmaf(cw[c], bf16lo(u.y), acc[2]); acc[3] = fmaf(cw[c], bf16hi(u.y), acc[3]);
          }
        }
      }
    }
  }
  out[q * rs + m * 8 + sub] = make_uint2(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]));
}

}  // namespace uc

using namespace uc;

extern "C" int uc_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                   const float* sampling_loc, const float* attn_weight, int B, int S, int M, int D, int L,
                                   int Lq, int P, float* out, void* stream_v) {
  if (!value || !spatial_shapes || !level_start_index || !sampling_loc || !attn_weight || !out)
    return set_error(UC_EINVAL, "uc_msda_forward_f32: null pointer");
  if (B <= 0 || S <= 0 || M <= 0 || D <= 0 || L <= 0 || Lq <= 0 || P <= 0) return set_error(UC_EINVAL, "uc_msda_forward_f32: bad sizes");
  const long total = static_cast<long>(B) * Lq * M * D;
  const int grid = static_cast<int>(std::min<long>((total + 255) / 256, static_cast<long>(num_sms()) * 32));
  launch_pdl(msda_f32_kernel, grid, 256, 0, static_cast<cudaStream_t>(stream_v), value, spatial_shapes, level_start_index, sampling_loc,
                                                                         attn_weight, out, B, S, M, D, L, Lq, P);
  return check_launch("uc_msda_forward_f32");
}

static int msda_fused(const char* what, const void* value, const float* offlog, int ld_offlog, void* out, const int* level_hw, int L,
                      int M, int P, int B, void* stream_v) {
  if (!value || !offlog || !out || !level_hw) return set_error(UC_EINVAL, "%s: null pointer", what);
  if (B < 1) return set_error(UC_EINVAL, "%s: B must be >= 1 (got %d)", what, B);
  if (L < 1 || L > 4 || L * P > 16 || M < 1) return set_error(UC_EINVAL, "%s: L<=4, L*P<=16 (head dim fixed at 32)", what);
  MsdaLevels lv;
  int start = 0;
  for (int l = 0; l < 4; ++l) {
    lv.H[l] = l < L ? level_hw[2 * l] : 1;
    lv.W[l] = l < L ? level_hw[2 * l + 1] : 1;
    lv.start[l] = start;
    if (l < L) start += lv.H[l] * lv.W[l];
  }
  const int Lq = start;
  const long threads = static_cast<long>(B) * Lq * M * 8;
  launch_pdl(msda_fused_kernel, static_cast<unsigned>((threads + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_v),
      static_cast<const uint2*>(value), offlog, static_cast<uint2*>(out), lv, M, L, P, Lq, ld_offlog, B);
  return check_launch(what);
}

extern "C" int uc_msda_fused_bf16(const void* value, const float* offlog, int ld_offlog, void* out, const int* level_hw, int L,
                                  int M, int P, void* stream_v) {
  return msda_fused("uc_msda_fused_bf16", value, offlog, ld_offlog, out, level_hw, L, M, P, 1, stream_v);
}

extern "C" int uc_msda_fused_bf16_batched(const void* value, const float* offlog, int ld_offlog, void* out, const int* level_hw, int L,
                                          int M, int P, int B, void* stream_v) {
  return msda_fused("uc_msda_fused_bf16_batched", value, offlog, ld_offlog, out, level_hw, L, M, P, B, stream_v);
}
